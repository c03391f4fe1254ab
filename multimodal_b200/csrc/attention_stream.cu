// Tensor-core self-attention for any sequence length, head_dim 64: the kernels attention.cu's entry points use for
// S > 384, where a whole head (Q, K, V and, backward, dO) no longer fits in shared memory.  Nothing in shared memory
// scales with S: each CTA keeps one 128-row block resident and streams the other operand through a ring of 64-row
// stages filled by cp.async, one mbarrier per stage (phase parity = use count & 1).  A stage is refilled only after
// the __syncthreads that opens the next iteration, i.e. once every warp has finished with it.
//
// Same arithmetic and layout contract as the resident kernels: packed qkv [B*S, 3*H*64] in, O bf16 [B*S, H*64] and
// lse fp32 [B, H, S] (natural log; optional) out, fp32 statistics, P and dS rounded to bf16 for the second product,
// exp2 with scale*log2(e), mma.sync m16n8k16 on ldmatrix fragments of XOR-swizzled tiles (attention_tiles.cuh).
//
//   attn_fwd_stream_kernel       grid (S/128, H, B); 8 warps x 16 query rows, Q fragments in registers, one
//                                online-softmax pass over 64-key blocks (causal: only blocks up to the diagonal).
//   attn_bwd_stream_dq_kernel    grid (S/128, H, B); D = rowsum(dO * O) of its rows -> scratch, then streams K / V to
//                                recompute S and dP and accumulates dQ = sum_j dS K.
//   attn_bwd_stream_dkdv_kernel  grid (S/128, H, B); 8 warps x 16 key rows, streams Q / dO (with their LSE and D) to
//                                form S^T and dP^T and accumulates dV = sum_i P^T dO and dK = sum_i dS^T Q.
// Every output element is owned by one warp and summed in a fixed order: no atomics, run-to-run deterministic.
// A row with no visible key gets O = 0 and lse = -inf, and contributes nothing to the backward; a masked key gets
// exactly zero dK and dV rows.
#include "attention_tiles.cuh"
#include "mmb200_internal.h"

namespace mmb {

constexpr int ST_BM = 128;               // rows a CTA owns (query rows, or key rows in the dK / dV kernel)
constexpr int ST_BN = 64;                // rows per streamed stage
constexpr int ST_THREADS = 256;          // 8 warps x 16 owned rows
constexpr int ST_CTAS_PER_SM = 2;        // launch bounds: 65536 / (2 * 256) = 128 registers per thread
constexpr int FWD_STAGES = 3;
constexpr int BWD_STAGES = 2;
constexpr int TILE_BYTES = ST_BN * 128;  // one 64-row x 64-column bf16 tile
constexpr float LOG2E = 1.4426950408889634f;

// rows [r0, r0 + n) of a strided bf16 matrix -> tile rows [0, n), asynchronously; rows >= S are zero-filled
__device__ __forceinline__ void cp_rows(uint8_t* dst, const __nv_bfloat16* src, long long ld, int S, int r0, int n) {
  for (int i = threadIdx.x; i < n * 8; i += blockDim.x) {
    const int r = i >> 3, ch = i & 7;
    const bool in = r0 + r < S;
    cp_async16(smem_u32(dst + toff(r, ch * 8)), src + (in ? (long long)(r0 + r) * ld + ch * 8 : 0), in ? 16u : 0u);
  }
}

// a warp's 16 x 64 fp32 accumulator tile (m16n8 fragments) -> bf16 rows [row0, row0 + 16) of a swizzled tile
__device__ __forceinline__ void frag_to_tile(uint8_t* tile, int row0, const float (&acc)[8][4], int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    *reinterpret_cast<uint32_t*>(tile + toff(row0 + g, nt * 8) + 4 * t) = pack_bf16x2(acc[nt][0], acc[nt][1]);
    *reinterpret_cast<uint32_t*>(tile + toff(row0 + g + 8, nt * 8) + 4 * t) = pack_bf16x2(acc[nt][2], acc[nt][3]);
  }
}
// tile rows [row0, row0 + 16) -> global rows grow0.. (< S) of a strided bf16 matrix, 16-byte stores
__device__ __forceinline__ void tile_to_global(__nv_bfloat16* dst, long long ld, const uint8_t* tile, int row0,
                                               int grow0, int S, int lane) {
  __syncwarp();
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int r = (it * 32 + lane) >> 3, ch = lane & 7;
    if (grow0 + r < S)
      *reinterpret_cast<uint4*>(dst + (long long)(grow0 + r) * ld + ch * 8) =
          *reinterpret_cast<const uint4*>(tile + toff(row0 + r, ch * 8));
  }
}

// LSE in log2 units for the backward; +inf for rows with no visible key (lse = -inf) and for padding rows, so that
// exp2(s - L) = 0 and such rows contribute nothing
__device__ __forceinline__ float lse_log2(const float* lse_row, int r, int S) {
  if (r >= S) return INFINITY;
  const float l = lse_row[r];
  return l == -INFINITY ? INFINITY : l * LOG2E;
}

// ------------------------------------------------------------------------------------------------
// Forward
// ------------------------------------------------------------------------------------------------
__host__ __device__ constexpr int fwd_stream_smem() {
  return ST_BM * 128 + 2 * FWD_STAGES * TILE_BYTES + 8 * FWD_STAGES + FWD_STAGES * ST_BN;
}

template <bool CAUSAL>
__global__ void __launch_bounds__(ST_THREADS, ST_CTAS_PER_SM) attn_fwd_stream_kernel(
    const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, float* __restrict__ lse,
    const uint8_t* __restrict__ kmask, int S, int H, float scale_log2) {
  extern __shared__ __align__(128) uint8_t asmem[];
  const int qb0 = blockIdx.x * ST_BM, h = blockIdx.y, b = blockIdx.z;
  const int d = H * HD;
  const long long ld = 3LL * d;
  uint8_t* sQ = asmem;                                                   // [128][64]
  uint8_t* sK = sQ + ST_BM * 128;                                        // [FWD_STAGES][64][64]
  uint8_t* sV = sK + FWD_STAGES * TILE_BYTES;                            // [FWD_STAGES][64][64]
  uint64_t* full = reinterpret_cast<uint64_t*>(sV + FWD_STAGES * TILE_BYTES);
  uint8_t* sM = reinterpret_cast<uint8_t*>(full + FWD_STAGES);           // [FWD_STAGES][64] key valid
  const __nv_bfloat16* base = qkv + (long long)b * S * ld + h * HD;
  const uint8_t* km = kmask ? kmask + (long long)b * S : nullptr;
  const int kv_end = CAUSAL ? min(S, qb0 + ST_BM) : S;
  const int n_kv = (kv_end + ST_BN - 1) / ST_BN;
  if (threadIdx.x == 0)
    for (int s = 0; s < FWD_STAGES; ++s) mbar_init(&full[s], blockDim.x);
  __syncthreads();
  // key block j -> stage j % FWD_STAGES: K, V and the key-valid flags (keys >= S are invalid)
  auto issue = [&](int j) {
    const int s = j % FWD_STAGES, k0 = j * ST_BN;
    cp_rows(sK + s * TILE_BYTES, base + d, ld, S, k0, ST_BN);
    cp_rows(sV + s * TILE_BYTES, base + 2 * d, ld, S, k0, ST_BN);
    if (threadIdx.x < ST_BN) {
      const int k = k0 + threadIdx.x;
      sM[s * ST_BN + threadIdx.x] = (k < S && (!km || km[k])) ? 1 : 0;
    }
    cp_async_arrive(&full[s]);
  };
  cp_rows(sQ, base, ld, S, qb0, ST_BM);   // completes with key block 0
  for (int j = 0; j < FWD_STAGES - 1 && j < n_kv; ++j) issue(j);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int q0 = qb0 + warp * 16;
  const int r0 = q0 + g, r1 = r0 + 8;
  const int w_end = CAUSAL ? min(kv_end, q0 + 16) : kv_end;   // keys this warp's rows can see
  uint32_t qa[4][4];
  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

#pragma unroll 1
  for (int j = 0; j < n_kv; ++j) {
    __syncthreads();   // every warp is done with block j - 1: its stage may be refilled
    if (j + FWD_STAGES - 1 < n_kv) issue(j + FWD_STAGES - 1);
    const int s = j % FWD_STAGES, kvb = j * ST_BN;
    mbar_wait_quiet(&full[s], (j / FWD_STAGES) & 1);
    if (j == 0) {
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) load_a(qa[ks], smem_u32(sQ), warp * 16, ks * 16, lane);
    }
    if (kvb >= w_end) continue;   // past this warp's diagonal
    const uint32_t uK = smem_u32(sK + s * TILE_BYTES), uV = smem_u32(sV + s * TILE_BYTES);
    const uint8_t* mk = sM + s * ST_BN;
    const int nt_valid = min(8, (w_end - kvb + 7) >> 3);
    float sc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
      if (nt < nt_valid) {
#pragma unroll
        for (int kp = 0; kp < 2; ++kp) {
          uint32_t kb[4];
          load_b_nk(kb, uK, nt * 8, kp * 32, lane);
          mma16816(sc[nt], qa[2 * kp], kb[0], kb[1]);
          mma16816(sc[nt], qa[2 * kp + 1], kb[2], kb[3]);
        }
      }
    }
    // per-element masking only where a key can be invalid: padded tail, key mask, causal diagonal
    const bool need_mask = km || kvb + ST_BN > S || (CAUSAL && kvb + ST_BN > q0);
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = sc[nt][e] * scale_log2;
        if (need_mask) {
          const int c = nt * 8 + 2 * t + (e & 1);
          const int row = (e < 2) ? r0 : r1;
          if (!mk[c] || (CAUSAL && kvb + c > row)) v = -INFINITY;
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
    for (int i = 0; i < 8; ++i) {
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
#pragma unroll
        for (int np = 0; np < 4; ++np) {
          uint32_t vb[4];
          load_b_kn(vb, uV, ks * 16, np * 16, lane);
          mma16816(o[2 * np], pa, vb[0], vb[1]);
          mma16816(o[2 * np + 1], pa, vb[2], vb[3]);
        }
      }
    }
  }
  l0 = quad_sum(l0);
  l1 = quad_sum(l1);
  const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    o[i][0] *= i0; o[i][1] *= i0; o[i][2] *= i1; o[i][3] *= i1;
  }
  // the warp's own 16 rows of sQ are free (its Q fragments are in registers): stage O there for 16-byte stores
  frag_to_tile(sQ, warp * 16, o, lane);
  tile_to_global(out + (long long)b * S * d + h * HD, d, sQ, warp * 16, q0, S, lane);
  if (lse && t == 0) {
    float* lrow = lse + ((long long)b * H + h) * S;
    if (r0 < S) lrow[r0] = (m0 + log2f(l0)) * 0.6931471805599453f;
    if (r1 < S) lrow[r1] = (m1 + log2f(l1)) * 0.6931471805599453f;
  }
}

// ------------------------------------------------------------------------------------------------
// Backward, launch 1: D and dQ for 128 query rows; K / V streamed in 64-key blocks
// ------------------------------------------------------------------------------------------------
__host__ __device__ constexpr int dq_stream_smem() {
  return 2 * ST_BM * 128 + 2 * BWD_STAGES * TILE_BYTES + ST_BM * 4 + 8 * BWD_STAGES + BWD_STAGES * ST_BN;
}

template <bool CAUSAL>
__global__ void __launch_bounds__(ST_THREADS, ST_CTAS_PER_SM) attn_bwd_stream_dq_kernel(
    const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ out,
    const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse, const uint8_t* __restrict__ kmask,
    __nv_bfloat16* __restrict__ dqkv, float* __restrict__ Dg, int S, int H, float scale) {
  extern __shared__ __align__(128) uint8_t asmem[];
  const int qb0 = blockIdx.x * ST_BM, h = blockIdx.y, b = blockIdx.z;
  const int d = H * HD;
  const long long ld = 3LL * d;
  uint8_t* sQ = asmem;                                                   // [128][64]
  uint8_t* sdO = sQ + ST_BM * 128;                                       // [128][64]
  uint8_t* sK = sdO + ST_BM * 128;                                       // [BWD_STAGES][64][64]
  uint8_t* sV = sK + BWD_STAGES * TILE_BYTES;                            // [BWD_STAGES][64][64]
  float* sD = reinterpret_cast<float*>(sV + BWD_STAGES * TILE_BYTES);   // [128] rowsum(dO * O)
  uint64_t* full = reinterpret_cast<uint64_t*>(sD + ST_BM);
  uint8_t* sM = reinterpret_cast<uint8_t*>(full + BWD_STAGES);           // [BWD_STAGES][64] key valid
  const long long bh = (long long)b * H + h;
  const __nv_bfloat16* base = qkv + (long long)b * S * ld + h * HD;
  const __nv_bfloat16* obase = out + (long long)b * S * d + h * HD;
  const __nv_bfloat16* dobase = dout + (long long)b * S * d + h * HD;
  const uint8_t* km = kmask ? kmask + (long long)b * S : nullptr;
  const int kv_end = CAUSAL ? min(S, qb0 + ST_BM) : S;
  const int n_kv = (kv_end + ST_BN - 1) / ST_BN;
  if (threadIdx.x == 0)
    for (int s = 0; s < BWD_STAGES; ++s) mbar_init(&full[s], blockDim.x);
  __syncthreads();
  auto issue = [&](int j) {
    const int s = j % BWD_STAGES, k0 = j * ST_BN;
    cp_rows(sK + s * TILE_BYTES, base + d, ld, S, k0, ST_BN);
    cp_rows(sV + s * TILE_BYTES, base + 2 * d, ld, S, k0, ST_BN);
    if (threadIdx.x < ST_BN) {
      const int k = k0 + threadIdx.x;
      sM[s * ST_BN + threadIdx.x] = (k < S && (!km || km[k])) ? 1 : 0;
    }
    cp_async_arrive(&full[s]);
  };
  cp_rows(sQ, base, ld, S, qb0, ST_BM);      // Q and dO complete with key block 0
  cp_rows(sdO, dobase, d, S, qb0, ST_BM);
  for (int j = 0; j < BWD_STAGES - 1 && j < n_kv; ++j) issue(j);
  // D = rowsum(dO * O) while the tiles land: eight lanes per row, one 16-byte chunk of O and of dO each
  for (int r = threadIdx.x >> 3; r < ST_BM; r += blockDim.x >> 3) {
    const int ch = threadIdx.x & 7, q = qb0 + r;
    float v = 0.f;
    if (q < S) {
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(obase + (long long)q * d + ch * 8));
      const uint4 c = __ldg(reinterpret_cast<const uint4*>(dobase + (long long)q * d + ch * 8));
      v = ((bf16_lo(a.x) * bf16_lo(c.x) + bf16_hi(a.x) * bf16_hi(c.x)) +
           (bf16_lo(a.y) * bf16_lo(c.y) + bf16_hi(a.y) * bf16_hi(c.y))) +
          ((bf16_lo(a.z) * bf16_lo(c.z) + bf16_hi(a.z) * bf16_hi(c.z)) +
           (bf16_lo(a.w) * bf16_lo(c.w) + bf16_hi(a.w) * bf16_hi(c.w)));
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (ch == 0) {
      sD[r] = v;
      if (q < S) Dg[bh * S + q] = v;
    }
  }

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int q0 = qb0 + warp * 16;
  const int r0 = q0 + g, r1 = r0 + 8;
  const int w_end = CAUSAL ? min(kv_end, q0 + 16) : kv_end;
  const float scale_log2 = scale * LOG2E;
  const float L0 = lse_log2(lse + bh * S, r0, S), L1 = lse_log2(lse + bh * S, r1, S);
  uint32_t qa[4][4], oa[4][4];
  float D0 = 0.f, D1 = 0.f;
  float dq[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) dq[n][0] = dq[n][1] = dq[n][2] = dq[n][3] = 0.f;

#pragma unroll 1
  for (int j = 0; j < n_kv; ++j) {
    __syncthreads();
    if (j + BWD_STAGES - 1 < n_kv) issue(j + BWD_STAGES - 1);
    const int s = j % BWD_STAGES, kvb = j * ST_BN;
    mbar_wait_quiet(&full[s], (j / BWD_STAGES) & 1);
    if (j == 0) {
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        load_a(qa[ks], smem_u32(sQ), warp * 16, ks * 16, lane);
        load_a(oa[ks], smem_u32(sdO), warp * 16, ks * 16, lane);
      }
      D0 = sD[warp * 16 + g];
      D1 = sD[warp * 16 + g + 8];
    }
    const uint32_t uK = smem_u32(sK + s * TILE_BYTES), uV = smem_u32(sV + s * TILE_BYTES);
    const uint8_t* mk = sM + s * ST_BN;
    const bool need_mask = km || kvb + ST_BN > S || (CAUSAL && kvb + ST_BN > q0);
#pragma unroll 1
    for (int kk = 0; kk < ST_BN / 16; ++kk) {
      const int kl = kk * 16;   // key offset within the block
      if (kvb + kl >= w_end) break;
      float sc[2][4], dp[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
        dp[nt][0] = dp[nt][1] = dp[nt][2] = dp[nt][3] = 0.f;
#pragma unroll
        for (int kp = 0; kp < 2; ++kp) {
          uint32_t kb[4], vb[4];
          load_b_nk(kb, uK, kl + nt * 8, kp * 32, lane);
          mma16816(sc[nt], qa[2 * kp], kb[0], kb[1]);
          mma16816(sc[nt], qa[2 * kp + 1], kb[2], kb[3]);
          load_b_nk(vb, uV, kl + nt * 8, kp * 32, lane);
          mma16816(dp[nt], oa[2 * kp], vb[0], vb[1]);
          mma16816(dp[nt], oa[2 * kp + 1], vb[2], vb[3]);
        }
      }
      uint32_t dsa[4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        float ds[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int c = kl + nt * 8 + 2 * t + (e & 1);
          bool valid = true;
          if (need_mask) valid = mk[c] && (!CAUSAL || kvb + c <= ((e < 2) ? r0 : r1));
          const float p = valid ? exp2f(sc[nt][e] * scale_log2 - ((e < 2) ? L0 : L1)) : 0.f;
          ds[e] = p * (dp[nt][e] - ((e < 2) ? D0 : D1)) * scale;
        }
        dsa[2 * nt] = pack_bf16x2(ds[0], ds[1]);
        dsa[2 * nt + 1] = pack_bf16x2(ds[2], ds[3]);
      }
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bb[4];
        load_b_kn(bb, uK, kl, np * 16, lane);
        mma16816(dq[2 * np], dsa, bb[0], bb[1]);
        mma16816(dq[2 * np + 1], dsa, bb[2], bb[3]);
      }
    }
  }
  frag_to_tile(sQ, warp * 16, dq, lane);
  tile_to_global(dqkv + (long long)b * S * ld + h * HD, ld, sQ, warp * 16, q0, S, lane);
}

// ------------------------------------------------------------------------------------------------
// Backward, launch 2: dK and dV for 128 key rows; Q / dO (with LSE and D) streamed in 64-query blocks
// ------------------------------------------------------------------------------------------------
__host__ __device__ constexpr int dkdv_stream_smem() {
  return 2 * ST_BM * 128 + 2 * BWD_STAGES * TILE_BYTES + 2 * BWD_STAGES * ST_BN * 4 + 8 * BWD_STAGES + ST_BM;
}

template <bool CAUSAL>
__global__ void __launch_bounds__(ST_THREADS, ST_CTAS_PER_SM) attn_bwd_stream_dkdv_kernel(
    const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse,
    const float* __restrict__ Dg, const uint8_t* __restrict__ kmask, __nv_bfloat16* __restrict__ dqkv, int S, int H,
    float scale) {
  extern __shared__ __align__(128) uint8_t asmem[];
  const int kb0 = blockIdx.x * ST_BM, h = blockIdx.y, b = blockIdx.z;
  const int d = H * HD;
  const long long ld = 3LL * d;
  uint8_t* sK = asmem;                                                   // [128][64]
  uint8_t* sV = sK + ST_BM * 128;                                        // [128][64]
  uint8_t* sQ = sV + ST_BM * 128;                                        // [BWD_STAGES][64][64]
  uint8_t* sdO = sQ + BWD_STAGES * TILE_BYTES;                           // [BWD_STAGES][64][64]
  float* sL = reinterpret_cast<float*>(sdO + BWD_STAGES * TILE_BYTES);  // [BWD_STAGES][64] LSE, log2 units
  float* sD = sL + BWD_STAGES * ST_BN;                                   // [BWD_STAGES][64] rowsum(dO * O)
  uint64_t* full = reinterpret_cast<uint64_t*>(sD + BWD_STAGES * ST_BN);
  uint8_t* sM = reinterpret_cast<uint8_t*>(full + BWD_STAGES);           // [128] key valid
  const int q_begin = CAUSAL ? kb0 : 0;   // causal: queries before the first key of the block see none of it
  const int n_q = (S - q_begin + ST_BN - 1) / ST_BN;
  if (threadIdx.x == 0)
    for (int s = 0; s < BWD_STAGES; ++s) mbar_init(&full[s], blockDim.x);
  for (int i = threadIdx.x; i < ST_BM; i += blockDim.x) {
    const int k = kb0 + i;
    sM[i] = (k < S && (!kmask || kmask[(long long)b * S + k])) ? 1 : 0;
  }
  __syncthreads();
  const __nv_bfloat16* base = qkv + (long long)b * S * ld + h * HD;
  const __nv_bfloat16* dobase = dout + (long long)b * S * d + h * HD;
  const float* lrow = lse + ((long long)b * H + h) * S;
  const float* drow = Dg + ((long long)b * H + h) * S;
  auto issue = [&](int j) {
    const int s = j % BWD_STAGES, qc = q_begin + j * ST_BN;
    cp_rows(sQ + s * TILE_BYTES, base, ld, S, qc, ST_BN);
    cp_rows(sdO + s * TILE_BYTES, dobase, d, S, qc, ST_BN);
    if (threadIdx.x < ST_BN) {
      sL[s * ST_BN + threadIdx.x] = lse_log2(lrow, qc + threadIdx.x, S);
    } else if (threadIdx.x < 2 * ST_BN) {
      const int q = qc + threadIdx.x - ST_BN;
      sD[s * ST_BN + threadIdx.x - ST_BN] = q < S ? drow[q] : 0.f;
    }
    cp_async_arrive(&full[s]);
  };
  cp_rows(sK, base + d, ld, S, kb0, ST_BM);   // K and V complete with query block 0
  cp_rows(sV, base + 2 * d, ld, S, kb0, ST_BM);
  for (int j = 0; j < BWD_STAGES - 1 && j < n_q; ++j) issue(j);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int kv0 = kb0 + warp * 16;
  const uint32_t uK = smem_u32(sK), uV = smem_u32(sV);
  const float scale_log2 = scale * LOG2E;
  float dk[8][4], dv[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
    dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
  }
  const bool keys_ok = __all_sync(0xffffffffu, sM[warp * 16 + g] && sM[warp * 16 + g + 8]);

#pragma unroll 1
  for (int j = 0; j < n_q; ++j) {
    __syncthreads();
    if (j + BWD_STAGES - 1 < n_q) issue(j + BWD_STAGES - 1);
    const int s = j % BWD_STAGES, qc = q_begin + j * ST_BN;
    mbar_wait_quiet(&full[s], (j / BWD_STAGES) & 1);
    const uint32_t uQ = smem_u32(sQ + s * TILE_BYTES), uO = smem_u32(sdO + s * TILE_BYTES);
    const float* L = sL + s * ST_BN;
    const float* Dq = sD + s * ST_BN;
#pragma unroll 1
    for (int qq = 0; qq < ST_BN / 16; ++qq) {
      const int ql = qq * 16, q0 = qc + ql;
      if (q0 >= S) break;
      if (CAUSAL && q0 + 16 <= kv0) continue;   // every query of the tile precedes every key of the warp
      // S^T = K Q^T -> P^T, which feeds dV before dP^T is formed (dK and dV hold 64 accumulator registers, so K and V
      // fragments are re-read from shared memory rather than kept)
      float p[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) p[nt][0] = p[nt][1] = p[nt][2] = p[nt][3] = 0.f;
#pragma unroll
      for (int kp = 0; kp < 2; ++kp) {
        uint32_t ka0[4], ka1[4];
        load_a(ka0, uK, warp * 16, kp * 32, lane);
        load_a(ka1, uK, warp * 16, kp * 32 + 16, lane);
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          uint32_t qb[4];
          load_b_nk(qb, uQ, ql + nt * 8, kp * 32, lane);
          mma16816(p[nt], ka0, qb[0], qb[1]);
          mma16816(p[nt], ka1, qb[2], qb[3]);
        }
      }
      const bool need_mask = !keys_ok || (CAUSAL && q0 < kv0 + 16);
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qi = ql + nt * 8 + 2 * t + (e & 1);
          bool valid = true;
          if (need_mask) valid = sM[warp * 16 + g + (e >> 1) * 8] && (!CAUSAL || kv0 + g + (e >> 1) * 8 <= qc + qi);
          p[nt][e] = valid ? exp2f(p[nt][e] * scale_log2 - L[qi]) : 0.f;
        }
      {
        uint32_t pa[4];
        pa[0] = pack_bf16x2(p[0][0], p[0][1]); pa[1] = pack_bf16x2(p[0][2], p[0][3]);
        pa[2] = pack_bf16x2(p[1][0], p[1][1]); pa[3] = pack_bf16x2(p[1][2], p[1][3]);
#pragma unroll
        for (int np = 0; np < 4; ++np) {
          uint32_t bb[4];
          load_b_kn(bb, uO, ql, np * 16, lane);
          mma16816(dv[2 * np], pa, bb[0], bb[1]);
          mma16816(dv[2 * np + 1], pa, bb[2], bb[3]);
        }
      }
      // dP^T = V dO^T -> dS^T = P^T (dP^T - D) * scale -> dK
      float dpt[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) dpt[nt][0] = dpt[nt][1] = dpt[nt][2] = dpt[nt][3] = 0.f;
#pragma unroll
      for (int kp = 0; kp < 2; ++kp) {
        uint32_t va0[4], va1[4];
        load_a(va0, uV, warp * 16, kp * 32, lane);
        load_a(va1, uV, warp * 16, kp * 32 + 16, lane);
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          uint32_t ob[4];
          load_b_nk(ob, uO, ql + nt * 8, kp * 32, lane);
          mma16816(dpt[nt], va0, ob[0], ob[1]);
          mma16816(dpt[nt], va1, ob[2], ob[3]);
        }
      }
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) dpt[nt][e] = p[nt][e] * (dpt[nt][e] - Dq[ql + nt * 8 + 2 * t + (e & 1)]) * scale;
      uint32_t dsa[4];
      dsa[0] = pack_bf16x2(dpt[0][0], dpt[0][1]); dsa[1] = pack_bf16x2(dpt[0][2], dpt[0][3]);
      dsa[2] = pack_bf16x2(dpt[1][0], dpt[1][1]); dsa[3] = pack_bf16x2(dpt[1][2], dpt[1][3]);
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bb[4];
        load_b_kn(bb, uQ, ql, np * 16, lane);
        mma16816(dk[2 * np], dsa, bb[0], bb[1]);
        mma16816(dk[2 * np + 1], dsa, bb[2], bb[3]);
      }
    }
  }
  // the warp's own rows of sK / sV are read by no other warp: stage dK / dV there for 16-byte stores
  __syncwarp();
  frag_to_tile(sK, warp * 16, dk, lane);
  frag_to_tile(sV, warp * 16, dv, lane);
  __nv_bfloat16* dbase = dqkv + (long long)b * S * ld + h * HD;
  tile_to_global(dbase + d, ld, sK, warp * 16, kv0, S, lane);
  tile_to_global(dbase + 2 * d, ld, sV, warp * 16, kv0, S, lane);
}

// ------------------------------------------------------------------------------------------------
// Launchers
// ------------------------------------------------------------------------------------------------
// grid.y = H and grid.z = B are limited to 65535
int attention_fwd_stream(const void* qkv, void* out, float* lse, const uint8_t* kmask, int B, int S, int H, int causal,
                         float scale, cudaStream_t st) {
  if (B > 65535 || H > 65535) return MMB_ERR_UNSUPPORTED;
  const int smem = fwd_stream_smem();
  auto kfn = causal ? attn_fwd_stream_kernel<true> : attn_fwd_stream_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return (int)e;
  const dim3 grid((S + ST_BM - 1) / ST_BM, H, B);
  kfn<<<grid, ST_THREADS, smem, st>>>((const __nv_bfloat16*)qkv, (__nv_bfloat16*)out, lse, kmask, S, H,
                                      scale * LOG2E);
  return (int)cudaGetLastError();
}

int attention_bwd_stream(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                         const uint8_t* kmask, int B, int S, int H, int causal, float scale, cudaStream_t st) {
  if (B > 65535 || H > 65535) return MMB_ERR_UNSUPPORTED;
  float* Dg = static_cast<float*>(scratch(SCR_ATTN_D, (size_t)B * H * S * sizeof(float), st));
  if (!Dg) return (int)cudaErrorMemoryAllocation;
  const dim3 grid((S + ST_BM - 1) / ST_BM, H, B);
  {
    const int smem = dq_stream_smem();
    auto kfn = causal ? attn_bwd_stream_dq_kernel<true> : attn_bwd_stream_dq_kernel<false>;
    cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    kfn<<<grid, ST_THREADS, smem, st>>>((const __nv_bfloat16*)qkv, (const __nv_bfloat16*)out,
                                        (const __nv_bfloat16*)dout, lse, kmask, (__nv_bfloat16*)dqkv, Dg, S, H, scale);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  }
  const int smem = dkdv_stream_smem();
  auto kfn = causal ? attn_bwd_stream_dkdv_kernel<true> : attn_bwd_stream_dkdv_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return (int)e;
  kfn<<<grid, ST_THREADS, smem, st>>>((const __nv_bfloat16*)qkv, (const __nv_bfloat16*)dout, lse, Dg, kmask,
                                      (__nv_bfloat16*)dqkv, S, H, scale);
  return (int)cudaGetLastError();
}

}  // namespace mmb
