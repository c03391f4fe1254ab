// Tensor-core attention with the general addressing of mmb_attention_fwd_generic / mmb_attention_bwd_generic
// (cross-attention, head_dim 64 / 96 / 128, batch-shared queries, [B, Sq, Skv] or key masks, top-left causal) for the
// shapes whose head does not fit in shared memory (generic_resident_fits() is false).  As in attention_stream.cu,
// nothing in shared memory grows with the sequence: a CTA keeps 128 rows resident and streams the other operand
// through a ring of 64-row stages filled by cp.async, one mbarrier per stage (phase parity = use count & 1).  A stage
// is refilled only after the __syncthreads that opens the next iteration, once every warp is done with it.
//
// Tiles are [rows][D] bf16 with a row pitch of 2*D + 16 bytes (an odd number of 16-byte chunks, so the 8 rows of an
// ldmatrix phase hit 8 distinct bank groups without a swizzle).  Operands are mma.sync m16n8k16 fragments read with
// ldmatrix; fp32 statistics, P and dS rounded to bf16 for the second product of each pair, exp2 with scale*log2(e).
// Masks are read from global memory per key block (mask[b*mask_bs + i*mask_qs + j], mask_qs = 0 for a key mask).
//
//   attn_fwd_gstream_kernel   grid (Sq/128, H, B); 8 warps x 16 query rows, one online-softmax pass over 64-key blocks
//                             (causal: only blocks up to the diagonal).  A row with no visible key gets O = 0.
//   attn_bwd_gstream_dq_kernel  grid (Sq/128, H, batch chunks); per batch two sweeps over K / V: the first forms the
//                             row LSE and D = sum_j p_ij dP_ij with online rescaling (written to the caller's scratch),
//                             the second accumulates dQ = sum_j dS_ij K_j.  Batch-shared queries: each CTA walks a
//                             chunk of the batch in order and keeps the chunk's fp32 sum in library scratch; a third
//                             kernel adds the chunks into dq_f32 in chunk order.
//   attn_bwd_gstream_dkdv_kernel  grid (Skv/128, H, B); 8 warps x 16 key rows, streams Q / dO with their LSE and D and
//                             accumulates dV = sum_i P^T dO and dK = sum_i dS^T Q.
// Every output element is owned by one warp and summed in a fixed order: no atomics, run-to-run deterministic, and the
// batch chunking depends only on the shape.  A masked key gets exactly zero dK and dV rows; a row with no visible key
// gets a zero dQ row.
#include "attention_generic.cuh"
#include "attention_tiles.cuh"
#include "mmb200_internal.h"

namespace mmb {

constexpr int GS_BM = 128;         // rows a CTA owns (query rows, or key rows in the dK / dV kernel)
constexpr int GS_BN = 64;          // rows per streamed stage
constexpr int GS_THREADS = 256;    // 8 warps x 16 owned rows
constexpr int GS_STAGES = 2;
// CTAs per SM each kernel's launch bounds plan, per head_dim (65536 / (GS_THREADS * ctas) registers per thread).  Two
// wherever the accumulators fit in 128 registers without spilling; one where they do not: the forward at D = 128 (64
// for O, 32 for S), dK / dV at D = 96 and 128 (dK + dV alone take D registers), and dQ at D = 128 (64 registers of dQ
// next to the S / dP tiles and their fragments: ptxas uses 196; its two resident 128-row tiles, 136 KB of shared
// memory, would also keep a second CTA off the SM).
constexpr int GS_FWD_CTAS_PER_SM_D64 = 2;
constexpr int GS_FWD_CTAS_PER_SM_D96 = 2;
constexpr int GS_FWD_CTAS_PER_SM_D128 = 1;
constexpr int GS_DQ_CTAS_PER_SM_D64 = 2;
constexpr int GS_DQ_CTAS_PER_SM_D96 = 2;
constexpr int GS_DQ_CTAS_PER_SM_D128 = 1;
constexpr int GS_DKDV_CTAS_PER_SM_D64 = 2;
constexpr int GS_DKDV_CTAS_PER_SM_D96 = 1;
constexpr int GS_DKDV_CTAS_PER_SM_D128 = 1;
// batch-shared queries: the batch is cut into chunks so that the dQ grid has about this many CTAs
constexpr int GS_DQ_TARGET_CTAS = 256;

template <int D> struct GsPlan;
template <> struct GsPlan<64> {
  static constexpr int fwd = GS_FWD_CTAS_PER_SM_D64, dq = GS_DQ_CTAS_PER_SM_D64, dkdv = GS_DKDV_CTAS_PER_SM_D64;
};
template <> struct GsPlan<96> {
  static constexpr int fwd = GS_FWD_CTAS_PER_SM_D96, dq = GS_DQ_CTAS_PER_SM_D96, dkdv = GS_DKDV_CTAS_PER_SM_D96;
};
template <> struct GsPlan<128> {
  static constexpr int fwd = GS_FWD_CTAS_PER_SM_D128, dq = GS_DQ_CTAS_PER_SM_D128, dkdv = GS_DKDV_CTAS_PER_SM_D128;
};

namespace gs {

template <int D> constexpr int pitch() { return 2 * D + 16; }

// A fragment (16 rows x 16 k) at rows r0.., cols c0.. of a row-major tile
template <int D>
__device__ __forceinline__ void load_a(uint32_t (&a)[4], uint32_t base, int r0, int c0, int lane) {
  ldsm_x4(a, base + (r0 + (lane & 7) + ((lane >> 3) & 1) * 8) * pitch<D>() + (c0 + (lane >> 4) * 8) * 2);
}
// B fragments from a tile stored [n][k]: 8 n-rows at n0, 32 k at k0 -> {b0,b1} for k-step k0 and k0+16
template <int D>
__device__ __forceinline__ void load_b_nk(uint32_t (&b)[4], uint32_t base, int n0, int k0, int lane) {
  ldsm_x4(b, base + (n0 + (lane & 7)) * pitch<D>() + (k0 + (lane >> 3) * 8) * 2);
}
// B fragments from a tile stored [k][n]: 16 k-rows at k0, 16 n at n0 -> {b0,b1} for n-tile n0 and n0+8
template <int D>
__device__ __forceinline__ void load_b_kn(uint32_t (&b)[4], uint32_t base, int k0, int n0, int lane) {
  ldsm_x4_t(b, base + (k0 + (lane & 7) + ((lane >> 3) & 1) * 8) * pitch<D>() + (n0 + (lane >> 4) * 8) * 2);
}

// rows [r0, r0 + n) of a strided bf16 matrix -> tile rows [0, n), asynchronously; rows >= S are zero-filled
template <int D>
__device__ __forceinline__ void cp_rows(uint8_t* dst, const __nv_bfloat16* src, long long ld, int S, int r0, int n) {
  constexpr int CH = D / 8;
  for (int i = threadIdx.x; i < n * CH; i += blockDim.x) {
    const int r = i / CH, ch = i - r * CH;
    const bool in = r0 + r < S;
    cp_async16(smem_u32(dst + r * pitch<D>() + ch * 16), src + (in ? (long long)(r0 + r) * ld + ch * 8 : 0),
               in ? 16u : 0u);
  }
}

// a warp's 16 x D fp32 accumulator tile -> bf16 rows [row0, row0 + 16) of a tile
template <int D>
__device__ __forceinline__ void frag_to_tile(uint8_t* tile, int row0, const float (&acc)[D / 8][4], int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int nt = 0; nt < D / 8; ++nt) {
    *reinterpret_cast<uint32_t*>(tile + (row0 + g) * pitch<D>() + (nt * 8 + 2 * t) * 2) = pack_bf16x2(acc[nt][0], acc[nt][1]);
    *reinterpret_cast<uint32_t*>(tile + (row0 + g + 8) * pitch<D>() + (nt * 8 + 2 * t) * 2) =
        pack_bf16x2(acc[nt][2], acc[nt][3]);
  }
}
// tile rows [row0, row0 + 16) -> global rows grow0.. (< S) of a strided bf16 matrix, 16-byte stores
template <int D>
__device__ __forceinline__ void tile_to_global(__nv_bfloat16* dst, long long ld, const uint8_t* tile, int row0,
                                               int grow0, int S, int lane) {
  constexpr int CH = D / 8;
  __syncwarp();
#pragma unroll
  for (int it = 0; it < D / 16; ++it) {
    const int idx = it * 32 + lane, r = idx / CH, ch = idx - r * CH;
    if (grow0 + r < S)
      *reinterpret_cast<uint4*>(dst + (long long)(grow0 + r) * ld + ch * 8) =
          *reinterpret_cast<const uint4*>(tile + (row0 + r) * pitch<D>() + ch * 16);
  }
}

// S (or S^T) tile of 16 rows x 16 columns: A rows from `ua` at ra, B rows (n) from `ub` at nb, over all D
template <int D>
__device__ __forceinline__ void product16(float (&acc)[2][4], uint32_t ua, int ra, uint32_t ub, int nb, int lane) {
#pragma unroll
  for (int nt = 0; nt < 2; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll
  for (int kp = 0; kp < D / 32; ++kp) {
    uint32_t a0[4], a1[4];
    load_a<D>(a0, ua, ra, kp * 32, lane);
    load_a<D>(a1, ua, ra, kp * 32 + 16, lane);
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      uint32_t b[4];
      load_b_nk<D>(b, ub, nb + nt * 8, kp * 32, lane);
      mma16816(acc[nt], a0, b[0], b[1]);
      mma16816(acc[nt], a1, b[2], b[3]);
    }
  }
}

// acc[16 x D] += A (16 x 16 bf16 fragment) * tile rows [k0, k0 + 16) (stored [k][n])
template <int D>
__device__ __forceinline__ void accum_pv(float (&acc)[D / 8][4], const uint32_t (&a)[4], uint32_t ub, int k0, int lane) {
#pragma unroll
  for (int np = 0; np < D / 16; ++np) {
    uint32_t b[4];
    load_b_kn<D>(b, ub, k0, np * 16, lane);
    mma16816(acc[2 * np], a, b[0], b[1]);
    mma16816(acc[2 * np + 1], a, b[2], b[3]);
  }
}

__device__ __forceinline__ bool visible(const uint8_t* mrow, int causal, int i, int j, int Skv) {
  return j < Skv && !(causal && j > i) && (!mrow || mrow[j]);
}

}  // namespace gs

// ------------------------------------------------------------------------------------------------
// Forward
// ------------------------------------------------------------------------------------------------
template <int D>
__host__ __device__ constexpr int gs_fwd_smem() {
  return (GS_BM + 2 * GS_STAGES * GS_BN) * gs::pitch<D>() + 8 * GS_STAGES;
}

template <int D, bool CAUSAL>
__global__ void __launch_bounds__(GS_THREADS, GsPlan<D>::fwd) attn_fwd_gstream_kernel(const AttnGenArgs p) {
  constexpr int P = gs::pitch<D>(), TILE = GS_BN * P, NO = D / 8;
  extern __shared__ __align__(128) uint8_t gsmem[];
  const int qb0 = blockIdx.x * GS_BM, h = blockIdx.y, b = blockIdx.z;
  uint8_t* sQ = gsmem;                                                   // [128][P]
  uint8_t* sK = sQ + GS_BM * P;                                          // [GS_STAGES][64][P]
  uint8_t* sV = sK + GS_STAGES * TILE;                                   // [GS_STAGES][64][P]
  uint64_t* full = reinterpret_cast<uint64_t*>(sV + GS_STAGES * TILE);
  const __nv_bfloat16* gq = p.q + b * p.bsq + h * D;
  const __nv_bfloat16* gk = p.k + b * p.bsk + h * D;
  const __nv_bfloat16* gv = p.v + b * p.bsv + h * D;
  const int kv_end = CAUSAL ? min(p.Skv, qb0 + GS_BM) : p.Skv;
  const int n_kv = (kv_end + GS_BN - 1) / GS_BN;
  if (threadIdx.x == 0)
    for (int s = 0; s < GS_STAGES; ++s) mbar_init(&full[s], blockDim.x);
  __syncthreads();
  auto issue = [&](int j) {
    const int s = j % GS_STAGES;
    gs::cp_rows<D>(sK + s * TILE, gk, p.ldk, p.Skv, j * GS_BN, GS_BN);
    gs::cp_rows<D>(sV + s * TILE, gv, p.ldv, p.Skv, j * GS_BN, GS_BN);
    cp_async_arrive(&full[s]);
  };
  gs::cp_rows<D>(sQ, gq, p.ldq, p.Sq, qb0, GS_BM);   // completes with key block 0
  for (int j = 0; j < GS_STAGES - 1 && j < n_kv; ++j) issue(j);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int q0 = qb0 + warp * 16;
  const int r0 = q0 + g, r1 = r0 + 8;
  // keys this warp's rows can see; none for a warp past the last query row
  const int w_end = q0 >= p.Sq ? 0 : (CAUSAL ? min(kv_end, q0 + 16) : kv_end);
  const uint8_t* mrow0 = p.mask ? p.mask + b * p.mask_bs + (long long)min(r0, p.Sq - 1) * p.mask_qs : nullptr;
  const uint8_t* mrow1 = p.mask ? p.mask + b * p.mask_bs + (long long)min(r1, p.Sq - 1) * p.mask_qs : nullptr;
  const uint32_t uQ = smem_u32(sQ);
  float o[NO][4];
#pragma unroll
  for (int i = 0; i < NO; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

#pragma unroll 1
  for (int j = 0; j < n_kv; ++j) {
    __syncthreads();   // every warp is done with block j - 1: its stage may be refilled
    if (j + GS_STAGES - 1 < n_kv) issue(j + GS_STAGES - 1);
    const int s = j % GS_STAGES, kvb = j * GS_BN;
    mbar_wait_quiet(&full[s], (j / GS_STAGES) & 1);
    if (kvb >= w_end) continue;   // past this warp's diagonal or its rows
    const uint32_t uK = smem_u32(sK + s * TILE), uV = smem_u32(sV + s * TILE);
    const int nt_valid = min(8, (w_end - kvb + 7) >> 3);
    float sc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
#pragma unroll
    for (int kp = 0; kp < D / 32; ++kp) {
      uint32_t qa0[4], qa1[4];
      gs::load_a<D>(qa0, uQ, warp * 16, kp * 32, lane);
      gs::load_a<D>(qa1, uQ, warp * 16, kp * 32 + 16, lane);
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        if (nt < nt_valid) {
          uint32_t kb[4];
          gs::load_b_nk<D>(kb, uK, nt * 8, kp * 32, lane);
          mma16816(sc[nt], qa0, kb[0], kb[1]);
          mma16816(sc[nt], qa1, kb[2], kb[3]);
        }
      }
    }
    // per-element masking only where a key can be invalid: padded tail, mask, causal diagonal
    const bool need_mask = p.mask || kvb + GS_BN > p.Skv || (CAUSAL && kvb + GS_BN > q0);
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = sc[nt][e] * p.scale_log2;
        if (need_mask) {
          const int c = kvb + nt * 8 + 2 * t + (e & 1);
          if (!gs::visible(e < 2 ? mrow0 : mrow1, CAUSAL, e < 2 ? r0 : r1, c, p.Skv)) v = -INFINITY;
        }
        sc[nt][e] = v;
      }
      mx0 = fmaxf(mx0, fmaxf(sc[nt][0], sc[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(sc[nt][2], sc[nt][3]));
    }
    mx0 = quad_max(mx0);
    mx1 = quad_max(mx1);
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    // rows with no valid key so far: subtract 0 (every exponent is 2^-inf = 0)
    const float b0 = (mn0 == -INFINITY) ? 0.f : mn0, b1 = (mn1 == -INFINITY) ? 0.f : mn1;
    const float c0 = exp2f(m0 - b0), c1 = exp2f(m1 - b1);
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      sc[nt][0] = exp2f(sc[nt][0] - b0);
      sc[nt][1] = exp2f(sc[nt][1] - b0);
      sc[nt][2] = exp2f(sc[nt][2] - b1);
      sc[nt][3] = exp2f(sc[nt][3] - b1);
      rs0 += sc[nt][0] + sc[nt][1];
      rs1 += sc[nt][2] + sc[nt][3];
    }
    l0 = l0 * c0 + rs0;
    l1 = l1 * c1 + rs1;
    m0 = mn0;
    m1 = mn1;
#pragma unroll
    for (int i = 0; i < NO; ++i) {
      o[i][0] *= c0; o[i][1] *= c0; o[i][2] *= c1; o[i][3] *= c1;
    }
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      if (2 * ks < nt_valid) {
        uint32_t pa[4];
        pa[0] = pack_bf16x2(sc[2 * ks][0], sc[2 * ks][1]);
        pa[1] = pack_bf16x2(sc[2 * ks][2], sc[2 * ks][3]);
        pa[2] = pack_bf16x2(sc[2 * ks + 1][0], sc[2 * ks + 1][1]);
        pa[3] = pack_bf16x2(sc[2 * ks + 1][2], sc[2 * ks + 1][3]);
        gs::accum_pv<D>(o, pa, uV, ks * 16, lane);
      }
    }
  }
  l0 = quad_sum(l0);
  l1 = quad_sum(l1);
  const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
#pragma unroll
  for (int i = 0; i < NO; ++i) {
    o[i][0] *= i0; o[i][1] *= i0; o[i][2] *= i1; o[i][3] *= i1;
  }
  // the warp's own 16 rows of sQ are read by no other warp: stage O there for 16-byte stores
  gs::frag_to_tile<D>(sQ, warp * 16, o, lane);
  gs::tile_to_global<D>(p.out + b * p.bso + h * D, p.ldo, sQ, warp * 16, q0, p.Sq, lane);
}

// ------------------------------------------------------------------------------------------------
// Backward, launch 1: LSE, D and dQ for 128 query rows; K / V streamed twice per batch in 64-key blocks
// ------------------------------------------------------------------------------------------------
template <int D>
__host__ __device__ constexpr int gs_dq_smem() {
  return (2 * GS_BM + 2 * GS_STAGES * GS_BN) * gs::pitch<D>() + 8 * GS_STAGES;
}

// part: fp32 [n_chunks][Sq][H*D] batch-chunk sums of dQ (dq_f32 requested), else unused; batches [z*per, z*per + per)
template <int D, bool CAUSAL>
__global__ void __launch_bounds__(GS_THREADS, GsPlan<D>::dq) attn_bwd_gstream_dq_kernel(const AttnGenBwdArgs p,
                                                                                       float* __restrict__ part,
                                                                                       int per) {
  constexpr int P = gs::pitch<D>(), TILE = GS_BN * P, NO = D / 8;
  extern __shared__ __align__(128) uint8_t gsmem[];
  const int qb0 = blockIdx.x * GS_BM, h = blockIdx.y;
  const int b_begin = blockIdx.z * per, b_end = min(p.B, b_begin + per);
  uint8_t* sQ = gsmem;                                                   // [128][P]
  uint8_t* sdO = sQ + GS_BM * P;                                         // [128][P]
  uint8_t* sK = sdO + GS_BM * P;                                         // [GS_STAGES][64][P]
  uint8_t* sV = sK + GS_STAGES * TILE;                                   // [GS_STAGES][64][P]
  uint64_t* full = reinterpret_cast<uint64_t*>(sV + GS_STAGES * TILE);
  const int kv_end = CAUSAL ? min(p.Skv, qb0 + GS_BM) : p.Skv;
  const int n_kv = (kv_end + GS_BN - 1) / GS_BN, n_it = 2 * n_kv;   // sweep 0: statistics, sweep 1: dQ
  if (threadIdx.x == 0)
    for (int s = 0; s < GS_STAGES; ++s) mbar_init(&full[s], blockDim.x);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int q0 = qb0 + warp * 16;
  const int r0 = q0 + g, r1 = r0 + 8;
  const int w_end = q0 >= p.Sq ? 0 : (CAUSAL ? min(kv_end, q0 + 16) : kv_end);
  const uint32_t uQ = smem_u32(sQ), uO = smem_u32(sdO);
  const int HD_all = p.H * D;

#pragma unroll 1
  for (int b = b_begin, it0 = 0; b < b_end; ++b, it0 += n_it) {
    const __nv_bfloat16* gq = p.q + b * p.bsq + h * D;
    const __nv_bfloat16* gdo = p.dout + b * p.bso + h * D;
    const __nv_bfloat16* gk = p.k + b * p.bsk + h * D;
    const __nv_bfloat16* gv = p.v + b * p.bsv + h * D;
    // ring use u (counted over the whole CTA) -> stage u % GS_STAGES, key block (u - it0) % n_kv
    auto issue = [&](int i) {
      const int u = it0 + i, s = u % GS_STAGES, k0 = (i % n_kv) * GS_BN;
      gs::cp_rows<D>(sK + s * TILE, gk, p.ldk, p.Skv, k0, GS_BN);
      gs::cp_rows<D>(sV + s * TILE, gv, p.ldv, p.Skv, k0, GS_BN);
      cp_async_arrive(&full[s]);
    };
    __syncthreads();   // the previous batch is done with sQ / sdO (and, first time round, the barriers are initialised)
    gs::cp_rows<D>(sQ, gq, p.ldq, p.Sq, qb0, GS_BM);   // Q and dO complete with the batch's first key block
    gs::cp_rows<D>(sdO, gdo, p.ldo, p.Sq, qb0, GS_BM);
    for (int i = 0; i < GS_STAGES - 1 && i < n_it; ++i) issue(i);

    const uint8_t* mrow0 = p.mask ? p.mask + b * p.mask_bs + (long long)min(r0, p.Sq - 1) * p.mask_qs : nullptr;
    const uint8_t* mrow1 = p.mask ? p.mask + b * p.mask_bs + (long long)min(r1, p.Sq - 1) * p.mask_qs : nullptr;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f, a0 = 0.f, a1 = 0.f;   // a: sum_j 2^(s_j - m) dP_j
    float L0 = INFINITY, L1 = INFINITY, D0 = 0.f, D1 = 0.f;
    float dq[NO][4];
#pragma unroll
    for (int i = 0; i < NO; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;

#pragma unroll 1
    for (int i = 0; i < n_it; ++i) {
      __syncthreads();
      if (i + GS_STAGES - 1 < n_it) issue(i + GS_STAGES - 1);
      const int u = it0 + i, s = u % GS_STAGES;
      const bool sweep_dq = i >= n_kv;
      const int kvb = (sweep_dq ? i - n_kv : i) * GS_BN;
      mbar_wait_quiet(&full[s], (u / GS_STAGES) & 1);
      if (i == n_kv) {   // statistics complete: log2-domain LSE (+inf for a row with no visible key) and D
        l0 = quad_sum(l0); l1 = quad_sum(l1);
        a0 = quad_sum(a0); a1 = quad_sum(a1);
        L0 = l0 > 0.f ? m0 + log2f(l0) : INFINITY;
        L1 = l1 > 0.f ? m1 + log2f(l1) : INFINITY;
        D0 = l0 > 0.f ? a0 / l0 : 0.f;
        D1 = l1 > 0.f ? a1 / l1 : 0.f;
        if (t == 0) {
          const long long row = ((long long)b * p.H + h) * p.Sq;
          if (r0 < p.Sq) { p.lse[row + r0] = L0; p.dsum[row + r0] = D0; }
          if (r1 < p.Sq) { p.lse[row + r1] = L1; p.dsum[row + r1] = D1; }
        }
      }
      const uint32_t uK = smem_u32(sK + s * TILE), uV = smem_u32(sV + s * TILE);
      const bool need_mask = p.mask || kvb + GS_BN > p.Skv || (CAUSAL && kvb + GS_BN > q0);
#pragma unroll 1
      for (int kk = 0; kk < GS_BN / 16; ++kk) {
        const int kl = kk * 16;   // key offset within the block
        if (kvb + kl >= w_end) break;
        float sc[2][4], dp[2][4];
        gs::product16<D>(sc, uQ, warp * 16, uK, kl, lane);
        gs::product16<D>(dp, uO, warp * 16, uV, kl, lane);
        auto ok = [&](int nt, int e) {
          return !need_mask || gs::visible(e < 2 ? mrow0 : mrow1, CAUSAL, e < 2 ? r0 : r1,
                                           kvb + kl + nt * 8 + 2 * t + (e & 1), p.Skv);
        };
        if (!sweep_dq) {
          float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
          for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              sc[nt][e] = ok(nt, e) ? sc[nt][e] * p.scale_log2 : -INFINITY;
              if (e < 2) mx0 = fmaxf(mx0, sc[nt][e]); else mx1 = fmaxf(mx1, sc[nt][e]);
            }
          mx0 = quad_max(mx0);
          mx1 = quad_max(mx1);
          const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
          const float b0 = (mn0 == -INFINITY) ? 0.f : mn0, b1 = (mn1 == -INFINITY) ? 0.f : mn1;
          const float c0 = exp2f(m0 - b0), c1 = exp2f(m1 - b1);
          l0 *= c0; a0 *= c0; l1 *= c1; a1 *= c1;
#pragma unroll
          for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float pe = exp2f(sc[nt][e] - (e < 2 ? b0 : b1));
              if (e < 2) { l0 += pe; a0 += pe * dp[nt][e]; } else { l1 += pe; a1 += pe * dp[nt][e]; }
            }
          m0 = mn0;
          m1 = mn1;
        } else {
          uint32_t dsa[4];
#pragma unroll
          for (int nt = 0; nt < 2; ++nt) {
            float ds[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float pe = ok(nt, e) ? exp2f(sc[nt][e] * p.scale_log2 - (e < 2 ? L0 : L1)) : 0.f;
              ds[e] = pe * (dp[nt][e] - (e < 2 ? D0 : D1)) * p.scale;
            }
            dsa[2 * nt] = pack_bf16x2(ds[0], ds[1]);
            dsa[2 * nt + 1] = pack_bf16x2(ds[2], ds[3]);
          }
          gs::accum_pv<D>(dq, dsa, uK, kl, lane);
        }
      }
    }
    if (p.dq) {   // the warp's own rows of sQ are read by no other warp
      gs::frag_to_tile<D>(sQ, warp * 16, dq, lane);
      gs::tile_to_global<D>(p.dq + b * p.bsq + h * D, p.ldq, sQ, warp * 16, q0, p.Sq, lane);
    }
    if (part) {   // this CTA owns these elements of its chunk's sum: add the batches in order
      float* prow0 = part + ((long long)blockIdx.z * p.Sq + r0) * HD_all + h * D;
      float* prow1 = part + ((long long)blockIdx.z * p.Sq + r1) * HD_all + h * D;
      const bool first = b == b_begin;
#pragma unroll
      for (int nt = 0; nt < NO; ++nt) {
        const int c = nt * 8 + 2 * t;
        if (r0 < p.Sq) {
          float2 v = make_float2(dq[nt][0], dq[nt][1]);
          if (!first) { const float2 o = *reinterpret_cast<float2*>(prow0 + c); v.x += o.x; v.y += o.y; }
          *reinterpret_cast<float2*>(prow0 + c) = v;
        }
        if (r1 < p.Sq) {
          float2 v = make_float2(dq[nt][2], dq[nt][3]);
          if (!first) { const float2 o = *reinterpret_cast<float2*>(prow1 + c); v.x += o.x; v.y += o.y; }
          *reinterpret_cast<float2*>(prow1 + c) = v;
        }
      }
    }
  }
}

// dq_f32[i, c] += sum_{z = 0..n_chunks-1} part[z, i, c], chunks in order
__global__ void __launch_bounds__(256) attn_bwd_gstream_dq_reduce_kernel(const float* __restrict__ part, int n_chunks,
                                                                         int Sq, int HD_all, float* __restrict__ dq_f32,
                                                                         long long ldq32) {
  const long long n = (long long)Sq * HD_all;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int z = 0; z < n_chunks; ++z) acc += part[z * n + idx];
    const long long i = idx / HD_all, c = idx - i * HD_all;
    dq_f32[i * ldq32 + c] += acc;
  }
}

// ------------------------------------------------------------------------------------------------
// Backward, launch 2: dK and dV for 128 key rows; Q / dO (with LSE and D) streamed in 64-query blocks
// ------------------------------------------------------------------------------------------------
template <int D>
__host__ __device__ constexpr int gs_dkdv_smem() {
  return (2 * GS_BM + 2 * GS_STAGES * GS_BN) * gs::pitch<D>() + 2 * GS_STAGES * GS_BN * 4 + 8 * GS_STAGES;
}

template <int D, bool CAUSAL>
__global__ void __launch_bounds__(GS_THREADS, GsPlan<D>::dkdv) attn_bwd_gstream_dkdv_kernel(const AttnGenBwdArgs p) {
  constexpr int P = gs::pitch<D>(), TILE = GS_BN * P, NO = D / 8;
  extern __shared__ __align__(128) uint8_t gsmem[];
  const int kb0 = blockIdx.x * GS_BM, h = blockIdx.y, b = blockIdx.z;
  uint8_t* sK = gsmem;                                                   // [128][P]
  uint8_t* sV = sK + GS_BM * P;                                          // [128][P]
  uint8_t* sQ = sV + GS_BM * P;                                          // [GS_STAGES][64][P]
  uint8_t* sdO = sQ + GS_STAGES * TILE;                                  // [GS_STAGES][64][P]
  float* sL = reinterpret_cast<float*>(sdO + GS_STAGES * TILE);          // [GS_STAGES][64] LSE, log2 units
  float* sD = sL + GS_STAGES * GS_BN;                                    // [GS_STAGES][64] D
  uint64_t* full = reinterpret_cast<uint64_t*>(sD + GS_STAGES * GS_BN);
  // causal (j <= i): queries before the first key of the block see none of it
  const int q_begin = CAUSAL ? kb0 : 0;
  const int n_q = q_begin >= p.Sq ? 0 : (p.Sq - q_begin + GS_BN - 1) / GS_BN;
  if (threadIdx.x == 0)
    for (int s = 0; s < GS_STAGES; ++s) mbar_init(&full[s], blockDim.x);
  __syncthreads();
  const __nv_bfloat16* gq = p.q + b * p.bsq + h * D;
  const __nv_bfloat16* gdo = p.dout + b * p.bso + h * D;
  const long long srow = ((long long)b * p.H + h) * p.Sq;
  auto issue = [&](int j) {
    const int s = j % GS_STAGES, qc = q_begin + j * GS_BN;
    gs::cp_rows<D>(sQ + s * TILE, gq, p.ldq, p.Sq, qc, GS_BN);
    gs::cp_rows<D>(sdO + s * TILE, gdo, p.ldo, p.Sq, qc, GS_BN);
    if (threadIdx.x < GS_BN) {
      const int q = qc + threadIdx.x;
      sL[s * GS_BN + threadIdx.x] = q < p.Sq ? p.lse[srow + q] : INFINITY;
    } else if (threadIdx.x < 2 * GS_BN) {
      const int q = qc + threadIdx.x - GS_BN;
      sD[s * GS_BN + threadIdx.x - GS_BN] = q < p.Sq ? p.dsum[srow + q] : 0.f;
    }
    cp_async_arrive(&full[s]);
  };
  gs::cp_rows<D>(sK, p.k + b * p.bsk + h * D, p.ldk, p.Skv, kb0, GS_BM);   // K and V complete with query block 0
  gs::cp_rows<D>(sV, p.v + b * p.bsv + h * D, p.ldv, p.Skv, kb0, GS_BM);
  for (int j = 0; j < GS_STAGES - 1 && j < n_q; ++j) issue(j);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int kv0 = kb0 + warp * 16;
  const uint32_t uK = smem_u32(sK), uV = smem_u32(sV);
  const uint8_t* mbase = p.mask ? p.mask + b * p.mask_bs : nullptr;
  float dk[NO][4], dv[NO][4];
#pragma unroll
  for (int i = 0; i < NO; ++i) {
    dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
    dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
  }

#pragma unroll 1
  for (int j = 0; j < n_q; ++j) {
    __syncthreads();
    if (j + GS_STAGES - 1 < n_q) issue(j + GS_STAGES - 1);
    const int s = j % GS_STAGES, qc = q_begin + j * GS_BN;
    mbar_wait_quiet(&full[s], (j / GS_STAGES) & 1);
    if (kv0 >= p.Skv) continue;   // no key row of this warp
    const uint32_t uQ = smem_u32(sQ + s * TILE), uO = smem_u32(sdO + s * TILE);
    const float* L = sL + s * GS_BN;
    const float* Dq = sD + s * GS_BN;
#pragma unroll 1
    for (int qq = 0; qq < GS_BN / 16; ++qq) {
      const int ql = qq * 16, q0 = qc + ql;
      if (q0 >= p.Sq) break;
      if (CAUSAL && q0 + 16 <= kv0) continue;   // every query of the tile precedes every key of the warp
      const bool need_mask = mbase || kv0 + 16 > p.Skv || q0 + 16 > p.Sq || (CAUSAL && q0 < kv0 + 16);
      // P^T = K Q^T, which feeds dV before dP^T is formed
      float pt[2][4];
      gs::product16<D>(pt, uK, warp * 16, uQ, ql, lane);
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qi = ql + nt * 8 + 2 * t + (e & 1), key = kv0 + g + (e >> 1) * 8, q = qc + qi;
          bool valid = true;
          if (need_mask)
            valid = key < p.Skv && q < p.Sq && !(CAUSAL && key > q) && (!mbase || mbase[(long long)q * p.mask_qs + key]);
          pt[nt][e] = valid ? exp2f(pt[nt][e] * p.scale_log2 - L[qi]) : 0.f;
        }
      {
        uint32_t pa[4];
        pa[0] = pack_bf16x2(pt[0][0], pt[0][1]); pa[1] = pack_bf16x2(pt[0][2], pt[0][3]);
        pa[2] = pack_bf16x2(pt[1][0], pt[1][1]); pa[3] = pack_bf16x2(pt[1][2], pt[1][3]);
        gs::accum_pv<D>(dv, pa, uO, ql, lane);
      }
      // dP^T = V dO^T -> dS^T = P^T (dP^T - D) * scale -> dK
      float dpt[2][4];
      gs::product16<D>(dpt, uV, warp * 16, uO, ql, lane);
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) dpt[nt][e] = pt[nt][e] * (dpt[nt][e] - Dq[ql + nt * 8 + 2 * t + (e & 1)]) * p.scale;
      uint32_t dsa[4];
      dsa[0] = pack_bf16x2(dpt[0][0], dpt[0][1]); dsa[1] = pack_bf16x2(dpt[0][2], dpt[0][3]);
      dsa[2] = pack_bf16x2(dpt[1][0], dpt[1][1]); dsa[3] = pack_bf16x2(dpt[1][2], dpt[1][3]);
      gs::accum_pv<D>(dk, dsa, uQ, ql, lane);
    }
  }
  // K / V may still be landing when no query block was streamed (causal, keys past the last query)
  cp_async_wait_all();
  __syncthreads();
  // the warp's own rows of sK / sV are read by no other warp: stage dK / dV there for 16-byte stores
  gs::frag_to_tile<D>(sK, warp * 16, dk, lane);
  gs::frag_to_tile<D>(sV, warp * 16, dv, lane);
  gs::tile_to_global<D>(p.dk + b * p.bsk + h * D, p.ldk, sK, warp * 16, kv0, p.Skv, lane);
  gs::tile_to_global<D>(p.dv + b * p.bsv + h * D, p.ldv, sV, warp * 16, kv0, p.Skv, lane);
}

// ------------------------------------------------------------------------------------------------
// Launchers
// ------------------------------------------------------------------------------------------------
template <typename K>
static int set_smem(K kfn, int smem) {
  return (int)cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
}

template <int D>
static int fwd_gstream(const AttnGenArgs& a, int B, cudaStream_t st) {
  const int smem = gs_fwd_smem<D>();
  auto kfn = a.causal ? attn_fwd_gstream_kernel<D, true> : attn_fwd_gstream_kernel<D, false>;
  if (int e = set_smem(kfn, smem)) return e;
  kfn<<<dim3((a.Sq + GS_BM - 1) / GS_BM, a.H, B), GS_THREADS, smem, st>>>(a);
  return (int)cudaGetLastError();
}

template <int D>
static int bwd_gstream(const AttnGenBwdArgs& a, cudaStream_t st) {
  const int n_qb = (a.Sq + GS_BM - 1) / GS_BM;
  // dq_f32: the batch is cut into chunks of `per` batches, a number that depends on the shape alone
  int per = 1, n_chunks = a.B;
  float* part = nullptr;
  if (a.dq_f32) {
    const int want = (GS_DQ_TARGET_CTAS + n_qb * a.H - 1) / (n_qb * a.H);
    n_chunks = want < 1 ? 1 : (want > a.B ? a.B : want);
    per = (a.B + n_chunks - 1) / n_chunks;
    n_chunks = (a.B + per - 1) / per;
    part = static_cast<float*>(scratch(SCR_ATTN_DQ, (size_t)n_chunks * a.Sq * a.H * D * sizeof(float), st));
    if (!part) return (int)cudaErrorMemoryAllocation;
  }
  {
    const int smem = gs_dq_smem<D>();
    auto kfn = a.causal ? attn_bwd_gstream_dq_kernel<D, true> : attn_bwd_gstream_dq_kernel<D, false>;
    if (int e = set_smem(kfn, smem)) return e;
    kfn<<<dim3(n_qb, a.H, n_chunks), GS_THREADS, smem, st>>>(a, part, per);
    if (int e = (int)cudaGetLastError()) return e;
  }
  {
    const int smem = gs_dkdv_smem<D>();
    auto kfn = a.causal ? attn_bwd_gstream_dkdv_kernel<D, true> : attn_bwd_gstream_dkdv_kernel<D, false>;
    if (int e = set_smem(kfn, smem)) return e;
    kfn<<<dim3((a.Skv + GS_BM - 1) / GS_BM, a.H, a.B), GS_THREADS, smem, st>>>(a);
    if (int e = (int)cudaGetLastError()) return e;
  }
  if (part) {
    const long long n = (long long)a.Sq * a.H * D;
    const int blocks = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
    attn_bwd_gstream_dq_reduce_kernel<<<blocks, 256, 0, st>>>(part, n_chunks, a.Sq, a.H * D, a.dq_f32, a.ldq32);
    return (int)cudaGetLastError();
  }
  return 0;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// cp.async reads and tile_to_global writes 16 bytes per row chunk: every operand and output base must be 16-byte aligned
int attention_fwd_gstream(const AttnGenArgs& a, int B, int D, cudaStream_t st) {
  if (!aligned16(a.q) || !aligned16(a.k) || !aligned16(a.v) || !aligned16(a.out)) return MMB_ERR_ARG;
  if (B > 65535 || a.H > 65535) return MMB_ERR_UNSUPPORTED;
  switch (D) {
    case 64: return fwd_gstream<64>(a, B, st);
    case 96: return fwd_gstream<96>(a, B, st);
    case 128: return fwd_gstream<128>(a, B, st);
    default: return MMB_ERR_UNSUPPORTED;
  }
}

int attention_bwd_gstream(const AttnGenBwdArgs& a, int D, cudaStream_t st) {
  if (!aligned16(a.q) || !aligned16(a.k) || !aligned16(a.v) || !aligned16(a.dout) || !aligned16(a.dk) ||
      !aligned16(a.dv) || (a.dq && !aligned16(a.dq)))
    return MMB_ERR_ARG;
  if (a.B > 65535 || a.H > 65535) return MMB_ERR_UNSUPPORTED;
  switch (D) {
    case 64: return bwd_gstream<64>(a, st);
    case 96: return bwd_gstream<96>(a, st);
    case 128: return bwd_gstream<128>(a, st);
    default: return MMB_ERR_UNSUPPORTED;
  }
}

}  // namespace mmb
