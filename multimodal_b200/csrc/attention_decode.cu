// Split-KV ("flash-decoding") attention for a few query rows over a long key / value cache, with the general addressing
// of mmb_attention_fwd_generic (row and batch strides, mask[b*mask_bs + i*mask_qs + j], top-left causal, head_dim 64 /
// 96 / 128), and the key / value cache concatenation of MultiHeadAttentionWithCache.
//
// At Sq <= 16 the general kernels use 16 of their 128 query rows and launch one CTA per (batch, head): at B = 1, H = 12
// that is 12 CTAs on 132 SMs, reading the cache with a tenth of the machine.  Here the keys are split across CTAs
// instead, and the partial results are combined in a fixed order:
//
//   attn_fwd_decode_kernel<D>   grid (splits, H, B), DEC_WARPS<D> warps.  A CTA owns a contiguous range of 64-key
//                               blocks; the query tile (one m16 tile, rows >= Sq masked) stays in registers.  Warp w takes
//                               blocks w, w + DEC_WARPS, ... of the range and streams them through its own ring of
//                               DEC_STAGES stages filled by cp.async, one mbarrier per stage (phase parity = use count
//                               & 1), keeping its own online-softmax state (m, l, O).  The warps merge through shared
//                               memory in warp order.  With one split the CTA writes bf16 O; otherwise it writes an fp32
//                               partial (unnormalised O, m, l) to library scratch (SCR_ATTN_DEC).  A split that lies
//                               wholly past the causal limit of the last query row writes an empty partial and loads
//                               nothing.
//   attn_decode_combine_kernel  adds the splits' partials in split order and writes bf16 O.  A row with no visible key
//                               gets O = 0, the convention of the general kernels.
//
// The split count depends only on (B, H, Skv) (decode_splits), never on the SM count, so results are the same run to
// run and card to card.  Roofline: 4 Sq Skv D flop against 4 Skv D bytes of K / V per head, at most 16 flop / byte at
// Sq = 16: the kernel is bound by HBM bandwidth.
//
//   kv_cache_append_kernel      out[b, s, h*hd + c] = s < Sp ? past[b, h, s, c] : new[b*Sn + s - Sp, h*hd + c]: torch.cat
//                               of a cache [B, H, Sp, hd] (fp32 or bf16, any B / H / S strides) and the new projection
//                               rows (bf16), into a fresh row-major [B, Sp + Sn, H*hd] buffer in the caller's dtype, plus
//                               the bf16 copy attention reads when that dtype is fp32.
#include "attention_generic.cuh"
#include "attention_tiles.cuh"
#include "mmb200_internal.h"

namespace mmb {

constexpr int DEC_BN = 64;              // keys per block
constexpr int DEC_STAGES = 2;           // ring stages per warp
constexpr int DEC_MAX_SQ = 16;          // one m16 query tile
// Splits: at least this many key blocks each, about this many CTAs in the grid, at most this many splits.  Constants,
// not the SM count, so that the split count (and with it the summation order) depends on the shape alone.
constexpr int DEC_MIN_BLOCKS_PER_SPLIT = 4;
constexpr int DEC_TARGET_CTAS = 264;
constexpr int DEC_MAX_SPLITS = 64;
// Warps per CTA and CTAs per SM each instantiation plans, per head_dim.  Shared memory decides: every warp owns
// DEC_STAGES stages of 64 K rows and 64 V rows at a pitch of 2*D + 16 bytes, i.e. 36.9 / 53.2 / 69.6 KB per warp at
// D = 64 / 96 / 128.  Four warps fit at D = 64 and 96 (147 / 213 KB), two at D = 128 (139 KB); one CTA per SM in each
// case, which keeps 8 / 8 / 4 blocks of K / V (147 / 213 / 139 KB) in flight per SM, far more than HBM latency needs.
constexpr int DEC_WARPS_D64 = 4;
constexpr int DEC_WARPS_D96 = 4;
constexpr int DEC_WARPS_D128 = 2;
constexpr int DEC_CTAS_PER_SM_D64 = 1;
constexpr int DEC_CTAS_PER_SM_D96 = 1;
constexpr int DEC_CTAS_PER_SM_D128 = 1;

template <int D> struct DecPlan;
template <> struct DecPlan<64> { static constexpr int warps = DEC_WARPS_D64, ctas = DEC_CTAS_PER_SM_D64; };
template <> struct DecPlan<96> { static constexpr int warps = DEC_WARPS_D96, ctas = DEC_CTAS_PER_SM_D96; };
template <> struct DecPlan<128> { static constexpr int warps = DEC_WARPS_D128, ctas = DEC_CTAS_PER_SM_D128; };

// Number of key splits for (B, H, Skv); every split holds at least one key block.
__host__ __device__ inline int decode_splits(int B, int H, int Skv) {
  const int nblk = (Skv + DEC_BN - 1) / DEC_BN;
  const long long bh = (long long)B * H;
  int n = (int)((DEC_TARGET_CTAS + bh - 1) / bh);
  const int by_len = nblk / DEC_MIN_BLOCKS_PER_SPLIT;
  if (n > by_len) n = by_len;
  if (n > DEC_MAX_SPLITS) n = DEC_MAX_SPLITS;
  if (n < 1) n = 1;
  const int per = (nblk + n - 1) / n;
  return (nblk + per - 1) / per;
}

namespace dec {

template <int D> constexpr int pitch() { return 2 * D + 16; }
template <int D> constexpr int tile_bytes() { return DEC_BN * pitch<D>(); }
// Merge area (aliases the rings once every warp is done): per warp 16 x D fp32 O at a row pitch of D + 4 floats, then
// 16 m and 16 l
template <int D> constexpr int merge_floats() { return 16 * (D + 4) + 32; }
template <int D>
__host__ __device__ constexpr int smem_bytes() {
  return 16 * pitch<D>() + DecPlan<D>::warps * (2 * DEC_STAGES * tile_bytes<D>() + 8 * DEC_STAGES);
}
static_assert(smem_bytes<96>() <= 227 * 1024 && smem_bytes<64>() <= 227 * 1024 && smem_bytes<128>() <= 227 * 1024,
              "decode kernel shared memory");
static_assert(DecPlan<64>::warps * 4 * merge_floats<64>() <= DecPlan<64>::warps * 2 * DEC_STAGES * tile_bytes<64>() &&
                  DecPlan<128>::warps * 4 * merge_floats<128>() <= DecPlan<128>::warps * 2 * DEC_STAGES * tile_bytes<128>(),
              "merge area fits in the rings");

// rows [r0, r0 + n) of a strided bf16 matrix -> tile rows [0, n), by the 32 lanes of one warp; rows >= S are zero-filled
template <int D>
__device__ __forceinline__ void cp_rows_warp(uint8_t* dst, const __nv_bfloat16* src, long long ld, int S, int r0, int n,
                                             int lane) {
  constexpr int CH = D / 8;
  for (int i = lane; i < n * CH; i += 32) {
    const int r = i / CH, ch = i - r * CH;
    const bool in = r0 + r < S;
    cp_async16(smem_u32(dst + r * pitch<D>() + ch * 16), src + (in ? (long long)(r0 + r) * ld + ch * 8 : 0),
               in ? 16u : 0u);
  }
}

template <int D>
__device__ __forceinline__ void load_a(uint32_t (&a)[4], uint32_t base, int r0, int c0, int lane) {
  ldsm_x4(a, base + (r0 + (lane & 7) + ((lane >> 3) & 1) * 8) * pitch<D>() + (c0 + (lane >> 4) * 8) * 2);
}
template <int D>
__device__ __forceinline__ void load_b_nk(uint32_t (&b)[4], uint32_t base, int n0, int k0, int lane) {
  ldsm_x4(b, base + (n0 + (lane & 7)) * pitch<D>() + (k0 + (lane >> 3) * 8) * 2);
}
template <int D>
__device__ __forceinline__ void load_b_kn(uint32_t (&b)[4], uint32_t base, int k0, int n0, int lane) {
  ldsm_x4_t(b, base + (k0 + (lane & 7) + ((lane >> 3) & 1) * 8) * pitch<D>() + (n0 + (lane >> 4) * 8) * 2);
}

__device__ __forceinline__ bool visible(const uint8_t* mrow, int causal, int i, int j, int Skv) {
  return j < Skv && !(causal && j > i) && (!mrow || mrow[j]);
}

}  // namespace dec

// part_o: fp32 [B*H][splits][16][D] unnormalised O; part_ml: fp32 [B*H][splits][16][2] {m (log2 units), l}
template <int D>
__global__ void __launch_bounds__(DecPlan<D>::warps * 32, DecPlan<D>::ctas)
    attn_fwd_decode_kernel(const AttnGenArgs p, int blocks_per_split, float* __restrict__ part_o,
                           float* __restrict__ part_ml) {
  constexpr int NW = DecPlan<D>::warps, P = dec::pitch<D>(), TILE = dec::tile_bytes<D>(), NO = D / 8, NQ = D / 16;
  constexpr int OP = D + 4;   // merge-area row pitch (floats)
  extern __shared__ __align__(128) uint8_t dsmem[];
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z, n_split = gridDim.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  uint8_t* sQ = dsmem;                                                              // [16][P]
  uint8_t* ring = sQ + 16 * P;                                                      // per warp: [STAGES][K|V][64][P]
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + NW * 2 * DEC_STAGES * TILE);  // per warp: [STAGES]
  uint8_t* wK = ring + warp * 2 * DEC_STAGES * TILE;
  uint64_t* full = bars + warp * DEC_STAGES;

  // keys every query row can see end at kv_end (causal: row Sq - 1 sees keys <= Sq - 1)
  const int kv_end = p.causal ? min(p.Skv, p.Sq) : p.Skv;
  const int blk0 = split * blocks_per_split;
  const int blk1 = min(blk0 + blocks_per_split, (kv_end + DEC_BN - 1) / DEC_BN);
  const int n_blk = max(0, blk1 - blk0);
  const long long bh = (long long)b * p.H + h;

  if (n_blk > 0) {
    const __nv_bfloat16* gk = p.k + b * p.bsk + h * D;
    const __nv_bfloat16* gv = p.v + b * p.bsv + h * D;
    // this warp's blocks: blk0 + warp + i * NW, i < n_w
    const int n_w = warp < n_blk ? (n_blk - warp + NW - 1) / NW : 0;
    if (lane == 0)
      for (int s = 0; s < DEC_STAGES; ++s) mbar_init(&full[s], 32);
    __syncwarp();
    auto issue = [&](int i) {
      const int s = i % DEC_STAGES, kb = (blk0 + warp + i * NW) * DEC_BN;
      dec::cp_rows_warp<D>(wK + (2 * s) * TILE, gk, p.ldk, p.Skv, kb, DEC_BN, lane);
      dec::cp_rows_warp<D>(wK + (2 * s + 1) * TILE, gv, p.ldv, p.Skv, kb, DEC_BN, lane);
      cp_async_arrive(&full[s]);
    };
    for (int i = 0; i < DEC_STAGES - 1 && i < n_w; ++i) issue(i);
    // the query tile: rows >= Sq are zero-filled
    for (int i = threadIdx.x; i < 16 * (D / 8); i += blockDim.x) {
      const int r = i / (D / 8), ch = i - r * (D / 8);
      uint4 v = make_uint4(0, 0, 0, 0);
      if (r < p.Sq) v = *reinterpret_cast<const uint4*>(p.q + b * p.bsq + (long long)r * p.ldq + h * D + ch * 8);
      *reinterpret_cast<uint4*>(sQ + r * P + ch * 16) = v;
    }
    __syncthreads();
    uint32_t qa[NQ][4];
#pragma unroll
    for (int kq = 0; kq < NQ; ++kq) dec::load_a<D>(qa[kq], smem_u32(sQ), 0, kq * 16, lane);

    const int r0 = g, r1 = g + 8;
    const uint8_t* mrow0 = p.mask ? p.mask + b * p.mask_bs + (long long)min(r0, p.Sq - 1) * p.mask_qs : nullptr;
    const uint8_t* mrow1 = p.mask ? p.mask + b * p.mask_bs + (long long)min(r1, p.Sq - 1) * p.mask_qs : nullptr;
    float o[NO][4];
#pragma unroll
    for (int i = 0; i < NO; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

#pragma unroll 1
    for (int i = 0; i < n_w; ++i) {
      __syncwarp();   // every lane is done with the stage block i - 1 used: it may be refilled
      if (i + DEC_STAGES - 1 < n_w) issue(i + DEC_STAGES - 1);
      const int s = i % DEC_STAGES, kvb = (blk0 + warp + i * NW) * DEC_BN;
      mbar_wait_quiet(&full[s], (i / DEC_STAGES) & 1);
      const uint32_t uK = smem_u32(wK + (2 * s) * TILE), uV = smem_u32(wK + (2 * s + 1) * TILE);
      const int nt_valid = min(8, (kv_end - kvb + 7) >> 3);
      float sc[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
#pragma unroll
      for (int kp = 0; kp < D / 32; ++kp) {
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          if (nt < nt_valid) {
            uint32_t kb[4];
            dec::load_b_nk<D>(kb, uK, nt * 8, kp * 32, lane);
            mma16816(sc[nt], qa[2 * kp], kb[0], kb[1]);
            mma16816(sc[nt], qa[2 * kp + 1], kb[2], kb[3]);
          }
        }
      }
      // per-element masking only where a key can be invalid: padded tail, mask, causal (rows >= Sq are zero queries
      // whose results are never written)
      const bool need_mask = p.mask || kvb + DEC_BN > p.Skv || p.causal;
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float v = sc[nt][e] * p.scale_log2;
          if (need_mask) {
            const int c = kvb + nt * 8 + 2 * t + (e & 1);
            if (!dec::visible(e < 2 ? mrow0 : mrow1, p.causal, e < 2 ? r0 : r1, c, p.Skv)) v = -INFINITY;
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
      for (int i2 = 0; i2 < NO; ++i2) {
        o[i2][0] *= c0; o[i2][1] *= c0; o[i2][2] *= c1; o[i2][3] *= c1;
      }
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        if (2 * ks < nt_valid) {
          uint32_t pa[4];
          pa[0] = pack_bf16x2(sc[2 * ks][0], sc[2 * ks][1]);
          pa[1] = pack_bf16x2(sc[2 * ks][2], sc[2 * ks][3]);
          pa[2] = pack_bf16x2(sc[2 * ks + 1][0], sc[2 * ks + 1][1]);
          pa[3] = pack_bf16x2(sc[2 * ks + 1][2], sc[2 * ks + 1][3]);
#pragma unroll
          for (int np = 0; np < D / 16; ++np) {
            uint32_t vb[4];
            dec::load_b_kn<D>(vb, uV, ks * 16, np * 16, lane);
            mma16816(o[2 * np], pa, vb[0], vb[1]);
            mma16816(o[2 * np + 1], pa, vb[2], vb[3]);
          }
        }
      }
    }
    l0 = quad_sum(l0);
    l1 = quad_sum(l1);
    __syncthreads();   // every warp is done with its ring (all of its cp.async copies were waited on): reuse it
    float* mo = reinterpret_cast<float*>(ring) + warp * dec::merge_floats<D>();
#pragma unroll
    for (int nt = 0; nt < NO; ++nt) {
      const int c = nt * 8 + 2 * t;
      *reinterpret_cast<float2*>(mo + r0 * OP + c) = make_float2(o[nt][0], o[nt][1]);
      *reinterpret_cast<float2*>(mo + r1 * OP + c) = make_float2(o[nt][2], o[nt][3]);
    }
    if (t == 0) {
      mo[16 * OP + r0] = m0; mo[16 * OP + 16 + r0] = l0;
      mo[16 * OP + r1] = m1; mo[16 * OP + 16 + r1] = l1;
    }
    __syncthreads();
    // merge the warps in warp order; a warp that had no block contributes m = -inf, l = 0, O = 0
    const float* mbase = reinterpret_cast<const float*>(ring);
    for (int idx = threadIdx.x; idx < 16 * D; idx += blockDim.x) {
      const int r = idx / D, c = idx - r * D;
      if (r >= p.Sq) continue;
      float M = -INFINITY;
#pragma unroll
      for (int w = 0; w < NW; ++w) M = fmaxf(M, mbase[w * dec::merge_floats<D>() + 16 * OP + r]);
      const float base = M == -INFINITY ? 0.f : M;
      float acc = 0.f, L = 0.f;
#pragma unroll
      for (int w = 0; w < NW; ++w) {
        const float* wm = mbase + w * dec::merge_floats<D>();
        const float f = exp2f(wm[16 * OP + r] - base);
        acc += wm[r * OP + c] * f;
        L += wm[16 * OP + 16 + r] * f;
      }
      if (n_split == 1) {
        p.out[b * p.bso + (long long)r * p.ldo + h * D + c] = __float2bfloat16_rn(L > 0.f ? acc / L : 0.f);
      } else {
        const long long prow = (bh * n_split + split) * 16 + r;
        part_o[prow * D + c] = acc;
        if (c == 0) { part_ml[prow * 2] = M; part_ml[prow * 2 + 1] = L; }
      }
    }
  } else {   // past the causal limit (so n_split > 1: split 0 always holds key 0): an empty partial, nothing loaded
    for (int idx = threadIdx.x; idx < 16 * D; idx += blockDim.x) {
      const int r = idx / D, c = idx - r * D;
      const long long prow = (bh * n_split + split) * 16 + r;
      part_o[prow * D + c] = 0.f;
      if (c == 0) { part_ml[prow * 2] = -INFINITY; part_ml[prow * 2 + 1] = 0.f; }
    }
  }
}

// O[b, r, h*D + c] = sum_s 2^(m_s - M) O_s / sum_s 2^(m_s - M) l_s, splits in order; 0 where no key is visible
__global__ void __launch_bounds__(128) attn_decode_combine_kernel(const float* __restrict__ part_o,
                                                                  const float* __restrict__ part_ml, int n_split, int D,
                                                                  int Sq, int H, __nv_bfloat16* __restrict__ out,
                                                                  long long ldo, long long bso) {
  const int h = blockIdx.y, b = blockIdx.z;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= Sq * D) return;
  const int r = idx / D, c = idx - r * D;
  const long long row0 = ((long long)b * H + h) * n_split * 16 + r;   // split s: row0 + s * 16
  float M = -INFINITY;
  for (int s = 0; s < n_split; ++s) M = fmaxf(M, part_ml[(row0 + s * 16) * 2]);
  const float base = M == -INFINITY ? 0.f : M;
  float acc = 0.f, L = 0.f;
  for (int s = 0; s < n_split; ++s) {
    const long long pr = row0 + s * 16;
    const float f = exp2f(part_ml[pr * 2] - base);
    acc += part_o[pr * D + c] * f;
    L += part_ml[pr * 2 + 1] * f;
  }
  out[b * bso + (long long)r * ldo + h * D + c] = __float2bfloat16_rn(L > 0.f ? acc / L : 0.f);
}

template <int D>
static int fwd_decode(const AttnGenArgs& a, int B, cudaStream_t st) {
  const int splits = decode_splits(B, a.H, a.Skv);
  const int nblk = (a.Skv + DEC_BN - 1) / DEC_BN;
  const int per = (nblk + splits - 1) / splits;
  float *part_o = nullptr, *part_ml = nullptr;
  if (splits > 1) {
    const size_t rows = (size_t)B * a.H * splits * 16;
    float* buf = static_cast<float*>(scratch(SCR_ATTN_DEC, rows * (D + 2) * sizeof(float), st));
    if (!buf) return (int)cudaErrorMemoryAllocation;
    part_o = buf;
    part_ml = buf + rows * D;
  }
  constexpr int smem = dec::smem_bytes<D>();
  auto kfn = attn_fwd_decode_kernel<D>;
  if (int e = (int)cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)) return e;
  kfn<<<dim3(splits, a.H, B), DecPlan<D>::warps * 32, smem, st>>>(a, per, part_o, part_ml);
  if (int e = (int)cudaGetLastError()) return e;
  if (splits > 1) {
    attn_decode_combine_kernel<<<dim3((a.Sq * D + 127) / 128, a.H, B), 128, 0, st>>>(part_o, part_ml, splits, D, a.Sq,
                                                                                     a.H, a.out, a.ldo, a.bso);
    return (int)cudaGetLastError();
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Key / value cache concatenation
// ------------------------------------------------------------------------------------------------
template <typename TP>
__global__ void __launch_bounds__(256) kv_cache_append_kernel(const TP* __restrict__ past, long long pbs, long long phs,
                                                              long long pss, const __nv_bfloat16* __restrict__ nw,
                                                              long long ld_new, void* __restrict__ out, int out_f32,
                                                              __nv_bfloat16* __restrict__ out_bf16, int H, int Sp, int Sn,
                                                              int hd, long long n) {
  const int HD = H * hd, St = Sp + Sn;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / HD;   // b * St + s
    const int col = (int)(i - row * HD);
    const int b = (int)(row / St), s = (int)(row - (long long)b * St);
    float v;
    if (s < Sp) {
      const int h = col / hd, c = col - h * hd;
      v = (float)past[b * pbs + h * phs + s * pss + c];
    } else {
      v = __bfloat162float(nw[((long long)b * Sn + (s - Sp)) * ld_new + col]);
    }
    if (out) {
      if (out_f32) static_cast<float*>(out)[i] = v;
      else static_cast<__nv_bfloat16*>(out)[i] = __float2bfloat16_rn(v);
    }
    if (out_bf16) out_bf16[i] = __float2bfloat16_rn(v);
  }
}

}  // namespace mmb

using namespace mmb;

extern "C" int mmb_attention_decode_splits(int B, int H, int Skv) {
  if (B <= 0 || H <= 0 || Skv <= 0) return MMB_ERR_ARG;
  return decode_splits(B, H, Skv);
}

static bool dec_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int mmb_attention_fwd_decode(const void* q, long long ldq, long long bsq, const void* k, long long ldk,
                                        long long bsk, const void* v, long long ldv, long long bsv, void* out,
                                        long long ldo, long long bso, const void* mask, long long mask_bs,
                                        long long mask_qs, int B, int Sq, int Skv, int H, int head_dim, int causal,
                                        float scale, void* stream) {
  if (B <= 0 || Sq <= 0 || Skv <= 0 || H <= 0) return MMB_ERR_ARG;
  if ((ldq | ldk | ldv | ldo | bsq | bsk | bsv | bso) & 7) return MMB_ERR_ARG;
  if (!dec_aligned16(q) || !dec_aligned16(k) || !dec_aligned16(v) || !dec_aligned16(out)) return MMB_ERR_ARG;
  if (Sq > DEC_MAX_SQ || (head_dim != 64 && head_dim != 96 && head_dim != 128)) return MMB_ERR_UNSUPPORTED;
  if (B > 65535 || H > 65535) return MMB_ERR_UNSUPPORTED;
  AttnGenArgs a{};
  a.q = (const __nv_bfloat16*)q; a.k = (const __nv_bfloat16*)k; a.v = (const __nv_bfloat16*)v;
  a.out = (__nv_bfloat16*)out;
  a.ldq = ldq; a.ldk = ldk; a.ldv = ldv; a.ldo = ldo; a.bsq = bsq; a.bsk = bsk; a.bsv = bsv; a.bso = bso;
  a.mask = (const uint8_t*)mask; a.mask_bs = mask_bs; a.mask_qs = mask_qs;
  a.Sq = Sq; a.Skv = Skv; a.H = H; a.causal = causal;
  a.scale_log2 = scale * 1.4426950408889634f;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (head_dim) {
    case 64: return fwd_decode<64>(a, B, st);
    case 96: return fwd_decode<96>(a, B, st);
    default: return fwd_decode<128>(a, B, st);
  }
}

extern "C" int mmb_kv_cache_append(const void* past, int past_f32, long long past_bs, long long past_hs,
                                   long long past_ss, const void* new_rows, long long ld_new, void* out, int out_f32,
                                   void* out_bf16, int B, int H, int Sp, int Sn, int head_dim, void* stream) {
  if (B <= 0 || H <= 0 || Sp < 0 || Sn < 0 || Sp + Sn <= 0 || head_dim <= 0) return MMB_ERR_ARG;
  if ((Sp > 0 && !past) || (Sn > 0 && !new_rows) || (!out && !out_bf16) || ld_new < (long long)H * head_dim)
    return MMB_ERR_ARG;
  const long long n = (long long)B * (Sp + Sn) * H * head_dim;
  long long blocks = (n + 255) / 256;
  if (blocks > 8192) blocks = 8192;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (past_f32)
    kv_cache_append_kernel<float><<<(int)blocks, 256, 0, st>>>(
        (const float*)past, past_bs, past_hs, past_ss, (const __nv_bfloat16*)new_rows, ld_new, out, out_f32,
        (__nv_bfloat16*)out_bf16, H, Sp, Sn, head_dim, n);
  else
    kv_cache_append_kernel<__nv_bfloat16><<<(int)blocks, 256, 0, st>>>(
        (const __nv_bfloat16*)past, past_bs, past_hs, past_ss, (const __nv_bfloat16*)new_rows, ld_new, out, out_f32,
        (__nv_bfloat16*)out_bf16, H, Sp, Sn, head_dim, n);
  return (int)cudaGetLastError();
}
