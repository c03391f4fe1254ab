// Tensor-core self-attention for S <= 384, head_dim 64 (CLIP ViT-B/16 image S = 197, text S = 77; ViT-L/14 S = 257;
// FLAVA; CoCa), one CTA per (batch, head).  The whole Q / K / V (and, backward, dO) of a head lives in shared memory
// (S = 384: 48 KB each), so each direction is a single pass: no split-KV, no second kernel, no scratch in HBM.  Operands
// are read straight out of the packed in-projection output [B*S, 3d] ([q | k | v], head h at columns h*64) and O is
// written as [B*S, d], the operand layout of the out-projection GEMM: no head split / merge copies.
// Replaces F.scaled_dot_product_attention + autograd (torch/nn/functional.py:6682).  Longer sequences go to the
// streamed kernels of attention_stream.cu through the same entry points.
//
// Math: softmax(Q K^T * scale) V with fp32 statistics; P (and dS) are rounded to bf16 for the second product.  Each warp
// owns 16-row tiles and runs m16n8k16 bf16 MMAs (fp32 accumulate) on fragments loaded with ldmatrix from XOR-swizzled
// shared tiles.  Optional key-padding mask [B,S] (1 = attend) and causal mask.
#include "attention_tiles.cuh"
#include "mmb200_internal.h"
#include <stdlib.h>

namespace mmb {

constexpr int SMAX = 384;

// cooperative load of rows [0,S) x 64 columns of a strided bf16 matrix into a swizzled tile; rows [S,S_pad) zeroed
__device__ __forceinline__ void load_tile(uint8_t* dst, const __nv_bfloat16* src, long long ld, int S, int S_pad) {
  for (int i = threadIdx.x; i < S_pad * 8; i += blockDim.x) {
    const int r = i >> 3, ch = i & 7;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r < S) v = __ldg(reinterpret_cast<const uint4*>(src + (long long)r * ld + ch * 8));
    *reinterpret_cast<uint4*>(dst + toff(r, ch * 8)) = v;
  }
}
// asynchronous form of load_tile for rows [r0, r1) (r1 <= S_pad); rows >= S are zero-filled
__device__ __forceinline__ void cp_tile_rows(uint8_t* dst, const __nv_bfloat16* src, long long ld, int S, int r0,
                                             int r1) {
  for (int i = r0 * 8 + threadIdx.x; i < r1 * 8; i += blockDim.x) {
    const int r = i >> 3, ch = i & 7;
    const bool in = r < S;
    cp_async16(smem_u32(dst + toff(r, ch * 8)), src + (in ? (long long)r * ld + ch * 8 : 0), in ? 16u : 0u);
  }
}

// key-valid flags: k < S and (no mask or mask[k] != 0)
__device__ __forceinline__ void load_keymask(uint8_t* dst, const uint8_t* kmask, int S, int S_pad) {
  for (int i = threadIdx.x; i < S_pad; i += blockDim.x) dst[i] = (i < S && (!kmask || kmask[i])) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------
// Forward
// ------------------------------------------------------------------------------------------------
template <bool CAUSAL>
__global__ void __launch_bounds__(256) attn_fwd_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                       __nv_bfloat16* __restrict__ out, float* __restrict__ lse,
                                                       const uint8_t* __restrict__ kmask, int S, int H,
                                                       float scale_log2) {
  extern __shared__ __align__(128) uint8_t asmem[];
  const int S_pad = (S + 15) & ~15;
  const int d = H * HD;
  const long long ld = 3LL * d;
  const int b = blockIdx.x / H, h = blockIdx.x - b * H;
  uint8_t* sQ = asmem;
  uint8_t* sK = sQ + S_pad * 128;
  uint8_t* sV = sK + S_pad * 128;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + S_pad * 128);  // [n_kc]: Q + keys 0..63, then 64 keys each
  uint8_t* sM = reinterpret_cast<uint8_t*>(bars + SMAX / 64);      // [S_pad] key valid
  const __nv_bfloat16* base = qkv + (long long)b * S * ld + h * HD;
  const int n_kc = (S_pad + 63) >> 6;
  if (threadIdx.x == 0)
    for (int c = 0; c < n_kc; ++c) mbar_init(&bars[c], blockDim.x);
  load_keymask(sM, kmask ? kmask + (long long)b * S : nullptr, S, S_pad);
  __syncthreads();
  // Q, then K and V in 64-key chunks in the order the key loop consumes them; chunk c completes bars[c]
  cp_tile_rows(sQ, base, ld, S, 0, S_pad);
  for (int c = 0; c < n_kc; ++c) {
    const int k1 = min(S_pad, (c + 1) * 64);
    cp_tile_rows(sK, base + d, ld, S, c * 64, k1);
    cp_tile_rows(sV, base + 2 * d, ld, S, c * 64, k1);
    cp_async_arrive(&bars[c]);
  }
  const uint32_t uQ = smem_u32(sQ), uK = smem_u32(sK), uV = smem_u32(sV);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int n_qt = S_pad >> 4;
  mbar_wait_quiet(&bars[0], 0);   // Q (and the first 64 keys)

  for (int qt = warp; qt < n_qt; qt += nwarps) {
    const int q0 = qt * 16;
    uint32_t qa[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) load_a(qa[ks], uQ, q0, ks * 16, lane);
    float o[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    const int r0 = q0 + g, r1 = r0 + 8;
    const int kv_end = CAUSAL ? min(S, q0 + 16) : S;

    for (int kvb = 0; kvb < kv_end; kvb += 64) {
      mbar_wait_quiet(&bars[kvb >> 6], 0);
      const int nt_valid = min(8, (kv_end - kvb + 7) >> 3);
      float s[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
        if (nt < nt_valid) {
#pragma unroll
          for (int kp = 0; kp < 2; ++kp) {
            uint32_t kb[4];
            load_b_nk(kb, uK, kvb + nt * 8, kp * 32, lane);
            mma16816(s[nt], qa[2 * kp], kb[0], kb[1]);
            mma16816(s[nt], qa[2 * kp + 1], kb[2], kb[3]);
          }
        }
      }
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int col = kvb + nt * 8 + 2 * t + (e & 1);
          const int row = (e < 2) ? r0 : r1;
          float v = s[nt][e] * scale_log2;
          if (col >= kv_end || !sM[col] || (CAUSAL && col > row)) v = -INFINITY;
          s[nt][e] = v;
        }
        mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
        mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
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
        s[nt][0] = exp2f(s[nt][0] - b0);
        s[nt][1] = exp2f(s[nt][1] - b0);
        s[nt][2] = exp2f(s[nt][2] - b1);
        s[nt][3] = exp2f(s[nt][3] - b1);
        rs0 += s[nt][0] + s[nt][1];
        rs1 += s[nt][2] + s[nt][3];
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
          pa[0] = pack_bf16x2(s[2 * ks][0], s[2 * ks][1]);
          pa[1] = pack_bf16x2(s[2 * ks][2], s[2 * ks][3]);
          pa[2] = pack_bf16x2(s[2 * ks + 1][0], s[2 * ks + 1][1]);
          pa[3] = pack_bf16x2(s[2 * ks + 1][2], s[2 * ks + 1][3]);
#pragma unroll
          for (int np = 0; np < 4; ++np) {
            uint32_t vb[4];
            load_b_kn(vb, uV, kvb + ks * 16, np * 16, lane);
            mma16816(o[2 * np], pa, vb[0], vb[1]);
            mma16816(o[2 * np + 1], pa, vb[2], vb[3]);
          }
        }
      }
    }
    l0 = quad_sum(l0);
    l1 = quad_sum(l1);
    // a row whose keys are all masked: O = 0, lse = -inf (its backward contributes nothing)
    const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
    __nv_bfloat16* orow0 = out + ((long long)b * S + r0) * d + h * HD;
    __nv_bfloat16* orow1 = out + ((long long)b * S + r1) * d + h * HD;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      if (r0 < S) *reinterpret_cast<uint32_t*>(orow0 + nt * 8 + 2 * t) = pack_bf16x2(o[nt][0] * i0, o[nt][1] * i0);
      if (r1 < S) *reinterpret_cast<uint32_t*>(orow1 + nt * 8 + 2 * t) = pack_bf16x2(o[nt][2] * i1, o[nt][3] * i1);
    }
    if (lse && t == 0) {
      float* lrow = lse + ((long long)b * H + h) * S;
      if (r0 < S) lrow[r0] = (m0 + log2f(l0)) * 0.6931471805599453f;
      if (r1 < S) lrow[r1] = (m1 + log2f(l1)) * 0.6931471805599453f;
    }
  }
  cp_async_wait_all();
}

// ------------------------------------------------------------------------------------------------
// Backward for S > BWD_STAGED_MAX, where dS does not fit in shared memory next to Q, K, V and dO.
//            Pass A: each warp owns 16 K/V rows and sweeps the query tiles -> dK, dV.
//            Pass B: each warp owns 16 query rows and sweeps the K/V tiles -> dQ (recomputes S and dP).
// D = rowsum(dO * O) is computed in the prologue.  No atomics, no cross-warp reductions, deterministic.
// ------------------------------------------------------------------------------------------------
template <bool CAUSAL>
__global__ void __launch_bounds__(256) attn_bwd_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                       const __nv_bfloat16* __restrict__ out,
                                                       const __nv_bfloat16* __restrict__ dout,
                                                       const float* __restrict__ lse,
                                                       const uint8_t* __restrict__ kmask,
                                                       __nv_bfloat16* __restrict__ dqkv, int S, int H, float scale) {
  extern __shared__ __align__(128) uint8_t asmem[];
  const int S_pad = (S + 15) & ~15;
  const int d = H * HD;
  const long long ld = 3LL * d;
  const int b = blockIdx.x / H, h = blockIdx.x - b * H;
  uint8_t* sQ = asmem;
  uint8_t* sK = sQ + S_pad * 128;
  uint8_t* sV = sK + S_pad * 128;
  uint8_t* sdO = sV + S_pad * 128;
  float* sL = reinterpret_cast<float*>(sdO + S_pad * 128);  // LSE in log2 units
  float* sD = sL + S_pad;                                   // rowsum(dO * O)
  uint8_t* sM = reinterpret_cast<uint8_t*>(sD + S_pad);     // [S_pad] key valid
  const __nv_bfloat16* base = qkv + (long long)b * S * ld + h * HD;
  const __nv_bfloat16* obase = out + (long long)b * S * d + h * HD;
  const __nv_bfloat16* dobase = dout + (long long)b * S * d + h * HD;
  load_tile(sQ, base, ld, S, S_pad);
  load_tile(sK, base + d, ld, S, S_pad);
  load_tile(sV, base + 2 * d, ld, S, S_pad);
  load_tile(sdO, dobase, d, S, S_pad);
  load_keymask(sM, kmask ? kmask + (long long)b * S : nullptr, S, S_pad);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int r = warp; r < S_pad; r += nwarps) {
    float acc = 0.f;
    if (r < S) {
      const uint32_t a = *reinterpret_cast<const uint32_t*>(obase + (long long)r * d + lane * 2);
      const uint32_t c = *reinterpret_cast<const uint32_t*>(dobase + (long long)r * d + lane * 2);
      acc = bf16_lo(a) * bf16_lo(c) + bf16_hi(a) * bf16_hi(c);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) {
      sD[r] = acc;
      sL[r] = (r < S) ? lse[((long long)b * H + h) * S + r] * 1.4426950408889634f : 0.f;
    }
  }
  __syncthreads();
  const uint32_t uQ = smem_u32(sQ), uK = smem_u32(sK), uV = smem_u32(sV), uO = smem_u32(sdO);
  const int g = lane >> 2, t = lane & 3;
  const int n_t = S_pad >> 4;
  const float scale_log2 = scale * 1.4426950408889634f;
  __nv_bfloat16* dbase = dqkv + (long long)b * S * ld + h * HD;

  // ---------------- Pass A: dK, dV ----------------
  for (int j = warp; j < n_t; j += nwarps) {
    const int kv0 = j * 16;
    uint32_t ka[4][4], va[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      load_a(ka[ks], uK, kv0, ks * 16, lane);
      load_a(va[ks], uV, kv0, ks * 16, lane);
    }
    float dk[8][4], dv[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
      dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
    }
    const bool kv_ok0 = sM[kv0 + g] != 0, kv_ok1 = sM[kv0 + g + 8] != 0;
    for (int i = CAUSAL ? j : 0; i < n_t; ++i) {
      const int q0 = i * 16;
      float st[2][4], dpt[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        st[nt][0] = st[nt][1] = st[nt][2] = st[nt][3] = 0.f;
        dpt[nt][0] = dpt[nt][1] = dpt[nt][2] = dpt[nt][3] = 0.f;
#pragma unroll
        for (int kp = 0; kp < 2; ++kp) {
          uint32_t qb[4], ob[4];
          load_b_nk(qb, uQ, q0 + nt * 8, kp * 32, lane);
          mma16816(st[nt], ka[2 * kp], qb[0], qb[1]);
          mma16816(st[nt], ka[2 * kp + 1], qb[2], qb[3]);
          load_b_nk(ob, uO, q0 + nt * 8, kp * 32, lane);
          mma16816(dpt[nt], va[2 * kp], ob[0], ob[1]);
          mma16816(dpt[nt], va[2 * kp + 1], ob[2], ob[3]);
        }
      }
      float pT[2][4], dsT[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int kv = kv0 + g + (e >> 1) * 8;
          const int q = q0 + nt * 8 + 2 * t + (e & 1);
          const bool valid = ((e >> 1) ? kv_ok1 : kv_ok0) && (q < S) && (!CAUSAL || kv <= q);
          const float p = valid ? exp2f(st[nt][e] * scale_log2 - sL[q]) : 0.f;
          pT[nt][e] = p;
          dsT[nt][e] = p * (dpt[nt][e] - sD[q]) * scale;
        }
      uint32_t pa[4], dsa[4];
      pa[0] = pack_bf16x2(pT[0][0], pT[0][1]); pa[1] = pack_bf16x2(pT[0][2], pT[0][3]);
      pa[2] = pack_bf16x2(pT[1][0], pT[1][1]); pa[3] = pack_bf16x2(pT[1][2], pT[1][3]);
      dsa[0] = pack_bf16x2(dsT[0][0], dsT[0][1]); dsa[1] = pack_bf16x2(dsT[0][2], dsT[0][3]);
      dsa[2] = pack_bf16x2(dsT[1][0], dsT[1][1]); dsa[3] = pack_bf16x2(dsT[1][2], dsT[1][3]);
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bb[4];
        load_b_kn(bb, uO, q0, np * 16, lane);
        mma16816(dv[2 * np], pa, bb[0], bb[1]);
        mma16816(dv[2 * np + 1], pa, bb[2], bb[3]);
        load_b_kn(bb, uQ, q0, np * 16, lane);
        mma16816(dk[2 * np], dsa, bb[0], bb[1]);
        mma16816(dk[2 * np + 1], dsa, bb[2], bb[3]);
      }
    }
    const int r0 = kv0 + g, r1 = r0 + 8;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      if (r0 < S) {
        *reinterpret_cast<uint32_t*>(dbase + (long long)r0 * ld + d + nt * 8 + 2 * t) = pack_bf16x2(dk[nt][0], dk[nt][1]);
        *reinterpret_cast<uint32_t*>(dbase + (long long)r0 * ld + 2 * d + nt * 8 + 2 * t) = pack_bf16x2(dv[nt][0], dv[nt][1]);
      }
      if (r1 < S) {
        *reinterpret_cast<uint32_t*>(dbase + (long long)r1 * ld + d + nt * 8 + 2 * t) = pack_bf16x2(dk[nt][2], dk[nt][3]);
        *reinterpret_cast<uint32_t*>(dbase + (long long)r1 * ld + 2 * d + nt * 8 + 2 * t) = pack_bf16x2(dv[nt][2], dv[nt][3]);
      }
    }
  }

  // ---------------- Pass B: dQ ----------------
  for (int i = warp; i < n_t; i += nwarps) {
    const int q0 = i * 16;
    uint32_t qa[4][4], oa[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      load_a(qa[ks], uQ, q0, ks * 16, lane);
      load_a(oa[ks], uO, q0, ks * 16, lane);
    }
    float dq[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) dq[n][0] = dq[n][1] = dq[n][2] = dq[n][3] = 0.f;
    const int r0 = q0 + g, r1 = r0 + 8;
    const float L0 = sL[r0], L1 = sL[r1], D0 = sD[r0], D1 = sD[r1];
    const int j_end = CAUSAL ? i + 1 : n_t;
    for (int j = 0; j < j_end; ++j) {
      const int kv0 = j * 16;
      float s[2][4], dp[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
        dp[nt][0] = dp[nt][1] = dp[nt][2] = dp[nt][3] = 0.f;
#pragma unroll
        for (int kp = 0; kp < 2; ++kp) {
          uint32_t kb[4], vb[4];
          load_b_nk(kb, uK, kv0 + nt * 8, kp * 32, lane);
          mma16816(s[nt], qa[2 * kp], kb[0], kb[1]);
          mma16816(s[nt], qa[2 * kp + 1], kb[2], kb[3]);
          load_b_nk(vb, uV, kv0 + nt * 8, kp * 32, lane);
          mma16816(dp[nt], oa[2 * kp], vb[0], vb[1]);
          mma16816(dp[nt], oa[2 * kp + 1], vb[2], vb[3]);
        }
      }
      float ds[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int row = (e < 2) ? r0 : r1;
          const int col = kv0 + nt * 8 + 2 * t + (e & 1);
          const bool valid = (row < S) && sM[col] && (!CAUSAL || col <= row);
          const float p = valid ? exp2f(s[nt][e] * scale_log2 - ((e < 2) ? L0 : L1)) : 0.f;
          ds[nt][e] = p * (dp[nt][e] - ((e < 2) ? D0 : D1)) * scale;
        }
      uint32_t dsa[4];
      dsa[0] = pack_bf16x2(ds[0][0], ds[0][1]); dsa[1] = pack_bf16x2(ds[0][2], ds[0][3]);
      dsa[2] = pack_bf16x2(ds[1][0], ds[1][1]); dsa[3] = pack_bf16x2(ds[1][2], ds[1][3]);
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bb[4];
        load_b_kn(bb, uK, kv0, np * 16, lane);
        mma16816(dq[2 * np], dsa, bb[0], bb[1]);
        mma16816(dq[2 * np + 1], dsa, bb[2], bb[3]);
      }
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      if (r0 < S) *reinterpret_cast<uint32_t*>(dbase + (long long)r0 * ld + nt * 8 + 2 * t) = pack_bf16x2(dq[nt][0], dq[nt][1]);
      if (r1 < S) *reinterpret_cast<uint32_t*>(dbase + (long long)r1 * ld + nt * 8 + 2 * t) = pack_bf16x2(dq[nt][2], dq[nt][3]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Backward with dS staged in shared memory (S_pad <= BWD_STAGED_MAX), five products instead of seven.
//   Pass A: warp j owns K/V rows [16j, 16j+16) and sweeps the query tiles in order -> dK, dV, and writes each bf16
//           dS^T(j, i) block it feeds to dK into sdS [kv][q].
//   Pass B: warp i owns query rows [16i, 16i+16) -> dQ(i) = sum_j dS(i, j) K(j), reading dS with transposing ldmatrix.
// The S^T / dP^T products of pass A are the S / dP products of the recompute kernel with the operands in swapped roles
// (same bf16 pairs, same k order), so dS, and with it dq / dk / dv, are the same bits.  One warp per 16-row tile.
// Loads are asynchronous and consumed in order: K and V complete bars[0], Q and dO rows [64c, 64c+64) bars[1 + c].
// ------------------------------------------------------------------------------------------------
constexpr int BWD_STAGED_MAX = 224;
constexpr int BWD_STAGED_THREADS = BWD_STAGED_MAX / 16 * 32;
constexpr int BWD_STAGED_BARS = 1 + (BWD_STAGED_MAX + 63) / 64;   // K and V, then one per 64 query rows

__host__ __device__ constexpr int ds_stride(int S_pad) { return 2 * S_pad + 16; }  // bytes; odd 16B units: no conflicts
__host__ __device__ constexpr int bwd_staged_smem(int S_pad) {
  return 4 * S_pad * 128 + S_pad * ds_stride(S_pad) + 2 * S_pad * 4 + 8 * BWD_STAGED_BARS + S_pad;
}
static_assert(bwd_staged_smem(BWD_STAGED_MAX) <= 227 * 1024, "staged backward exceeds the sm_90 shared-memory opt-in");

template <bool CAUSAL>
__global__ void __launch_bounds__(BWD_STAGED_THREADS, 1) attn_bwd_staged_kernel(
    const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout,
    const float* __restrict__ lse, const uint8_t* __restrict__ kmask, __nv_bfloat16* __restrict__ dqkv, int S, int H,
    float scale) {
  extern __shared__ __align__(128) uint8_t asmem[];
  const int S_pad = (S + 15) & ~15;
  const int dstride = ds_stride(S_pad);
  const int d = H * HD;
  const long long ld = 3LL * d;
  const int b = blockIdx.x / H, h = blockIdx.x - b * H;
  uint8_t* sQ = asmem;
  uint8_t* sK = sQ + S_pad * 128;
  uint8_t* sV = sK + S_pad * 128;
  uint8_t* sdO = sV + S_pad * 128;
  uint8_t* sdS = sdO + S_pad * 128;                                  // [S_pad kv][S_pad q] bf16, dstride bytes/row
  float* sL = reinterpret_cast<float*>(sdS + S_pad * dstride);      // LSE in log2 units
  float* sD = sL + S_pad;                                            // rowsum(dO * O)
  uint64_t* bars = reinterpret_cast<uint64_t*>(sD + S_pad);         // [BWD_STAGED_BARS]
  uint8_t* sM = reinterpret_cast<uint8_t*>(bars + BWD_STAGED_BARS);  // [S_pad] key valid
  const __nv_bfloat16* base = qkv + (long long)b * S * ld + h * HD;
  const __nv_bfloat16* obase = out + (long long)b * S * d + h * HD;
  const __nv_bfloat16* dobase = dout + (long long)b * S * d + h * HD;
  const int n_qc = (S_pad + 63) >> 6;
  if (threadIdx.x == 0)
    for (int c = 0; c <= n_qc; ++c) mbar_init(&bars[c], blockDim.x);
  load_keymask(sM, kmask ? kmask + (long long)b * S : nullptr, S, S_pad);
  __syncthreads();
  cp_tile_rows(sK, base + d, ld, S, 0, S_pad);
  cp_tile_rows(sV, base + 2 * d, ld, S, 0, S_pad);
  cp_async_arrive(&bars[0]);
  for (int c = 0; c < n_qc; ++c) {
    const int q1 = min(S_pad, (c + 1) * 64);
    cp_tile_rows(sQ, base, ld, S, c * 64, q1);
    cp_tile_rows(sdO, dobase, d, S, c * 64, q1);
    cp_async_arrive(&bars[1 + c]);
  }
  // D = rowsum(dO * O) while the tiles land: eight lanes per row, one 16-byte chunk of O and of dO each.  The sum runs
  // in the order of the recompute kernel's 32-lane butterfly over bf16 pairs (pair p = 4 * chunk + k): xor 16, 8, 4
  // across chunks (lane xor 4, 2, 1), then xor 2 and 1 within the chunk.
  for (int r = threadIdx.x >> 3; r < S_pad; r += blockDim.x >> 3) {
    const int ch = threadIdx.x & 7;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (r < S) {
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(obase + (long long)r * d + ch * 8));
      const uint4 c = __ldg(reinterpret_cast<const uint4*>(dobase + (long long)r * d + ch * 8));
      v[0] = bf16_lo(a.x) * bf16_lo(c.x) + bf16_hi(a.x) * bf16_hi(c.x);
      v[1] = bf16_lo(a.y) * bf16_lo(c.y) + bf16_hi(a.y) * bf16_hi(c.y);
      v[2] = bf16_lo(a.z) * bf16_lo(c.z) + bf16_hi(a.z) * bf16_hi(c.z);
      v[3] = bf16_lo(a.w) * bf16_lo(c.w) + bf16_hi(a.w) * bf16_hi(c.w);
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1)
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (ch == 0) {
      sD[r] = (v[0] + v[2]) + (v[1] + v[3]);
      sL[r] = (r < S) ? lse[((long long)b * H + h) * S + r] * 1.4426950408889634f : 0.f;
    }
  }
  __syncthreads();
  const uint32_t uQ = smem_u32(sQ), uK = smem_u32(sK), uV = smem_u32(sV), uO = smem_u32(sdO), udS = smem_u32(sdS);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int n_t = S_pad >> 4;
  const float scale_log2 = scale * 1.4426950408889634f;
  __nv_bfloat16* dbase = dqkv + (long long)b * S * ld + h * HD;

  // ---------------- Pass A: dK, dV, dS^T ----------------
  {
    const int j = warp, kv0 = j * 16;
    mbar_wait_quiet(&bars[0], 0);
    float dk[8][4], dv[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
      dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
    }
    const bool kv_ok0 = sM[kv0 + g] != 0, kv_ok1 = sM[kv0 + g + 8] != 0;
    const int i0 = CAUSAL ? j : 0;
#pragma unroll 1
    for (int i = i0; i < n_t; ++i) {
      // Q / dO rows of this chunk (one try_wait once they have landed)
      while (!mbar_try_wait(&bars[1 + (i >> 2)], 0)) {}
      const int q0 = i * 16;
      float st[2][4], dpt[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        st[nt][0] = st[nt][1] = st[nt][2] = st[nt][3] = 0.f;
        dpt[nt][0] = dpt[nt][1] = dpt[nt][2] = dpt[nt][3] = 0.f;
      }
      // K and V fragments are re-read from shared memory rather than held across the sweep: with 13-14 warps per
      // CTA, four share an SM sub-partition, which leaves 128 registers per thread
#pragma unroll
      for (int kp = 0; kp < 2; ++kp) {
        uint32_t ka0[4], ka1[4];
        load_a(ka0, uK, kv0, kp * 32, lane);
        load_a(ka1, uK, kv0, kp * 32 + 16, lane);
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          uint32_t qb[4];
          load_b_nk(qb, uQ, q0 + nt * 8, kp * 32, lane);
          mma16816(st[nt], ka0, qb[0], qb[1]);
          mma16816(st[nt], ka1, qb[2], qb[3]);
        }
      }
#pragma unroll
      for (int kp = 0; kp < 2; ++kp) {
        uint32_t va0[4], va1[4];
        load_a(va0, uV, kv0, kp * 32, lane);
        load_a(va1, uV, kv0, kp * 32 + 16, lane);
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          uint32_t ob[4];
          load_b_nk(ob, uO, q0 + nt * 8, kp * 32, lane);
          mma16816(dpt[nt], va0, ob[0], ob[1]);
          mma16816(dpt[nt], va1, ob[2], ob[3]);
        }
      }
      float pT[2][4], dsT[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int kv = kv0 + g + (e >> 1) * 8;
          const int q = q0 + nt * 8 + 2 * t + (e & 1);
          const bool valid = ((e >> 1) ? kv_ok1 : kv_ok0) && (q < S) && (!CAUSAL || kv <= q);
          const float p = valid ? exp2f(st[nt][e] * scale_log2 - sL[q]) : 0.f;
          pT[nt][e] = p;
          dsT[nt][e] = p * (dpt[nt][e] - sD[q]) * scale;
        }
      uint32_t pa[4], dsa[4];
      pa[0] = pack_bf16x2(pT[0][0], pT[0][1]); pa[1] = pack_bf16x2(pT[0][2], pT[0][3]);
      pa[2] = pack_bf16x2(pT[1][0], pT[1][1]); pa[3] = pack_bf16x2(pT[1][2], pT[1][3]);
      dsa[0] = pack_bf16x2(dsT[0][0], dsT[0][1]); dsa[1] = pack_bf16x2(dsT[0][2], dsT[0][3]);
      dsa[2] = pack_bf16x2(dsT[1][0], dsT[1][1]); dsa[3] = pack_bf16x2(dsT[1][2], dsT[1][3]);
      // dsa is the A fragment of dS^T(j, i): rows kv0 + g (+8), columns q0 + 2t (+8)
      uint8_t* ds_row0 = sdS + (kv0 + g) * dstride + (q0 + 2 * t) * 2;
      *reinterpret_cast<uint32_t*>(ds_row0) = dsa[0];
      *reinterpret_cast<uint32_t*>(ds_row0 + 8 * dstride) = dsa[1];
      *reinterpret_cast<uint32_t*>(ds_row0 + 16) = dsa[2];
      *reinterpret_cast<uint32_t*>(ds_row0 + 8 * dstride + 16) = dsa[3];
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bb[4];
        load_b_kn(bb, uO, q0, np * 16, lane);
        mma16816(dv[2 * np], pa, bb[0], bb[1]);
        mma16816(dv[2 * np + 1], pa, bb[2], bb[3]);
        load_b_kn(bb, uQ, q0, np * 16, lane);
        mma16816(dk[2 * np], dsa, bb[0], bb[1]);
        mma16816(dk[2 * np + 1], dsa, bb[2], bb[3]);
      }
    }
    const int r0 = kv0 + g, r1 = r0 + 8;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      if (r0 < S) {
        *reinterpret_cast<uint32_t*>(dbase + (long long)r0 * ld + d + nt * 8 + 2 * t) = pack_bf16x2(dk[nt][0], dk[nt][1]);
        *reinterpret_cast<uint32_t*>(dbase + (long long)r0 * ld + 2 * d + nt * 8 + 2 * t) = pack_bf16x2(dv[nt][0], dv[nt][1]);
      }
      if (r1 < S) {
        *reinterpret_cast<uint32_t*>(dbase + (long long)r1 * ld + d + nt * 8 + 2 * t) = pack_bf16x2(dk[nt][2], dk[nt][3]);
        *reinterpret_cast<uint32_t*>(dbase + (long long)r1 * ld + 2 * d + nt * 8 + 2 * t) = pack_bf16x2(dv[nt][2], dv[nt][3]);
      }
    }
  }
  cp_async_wait_all();
  __syncthreads();

  // ---------------- Pass B: dQ ----------------
  {
    const int i = warp, q0 = i * 16;
    float dq[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) dq[n][0] = dq[n][1] = dq[n][2] = dq[n][3] = 0.f;
    // lane -> row address of the transposed 8x8 blocks {q0, kv0}, {q0 + 8, kv0}, {q0, kv0 + 8}, {q0 + 8, kv0 + 8}
    const uint32_t ds_lane = udS + ((lane & 7) + ((lane >> 4) & 1) * 8) * dstride + (q0 + ((lane >> 3) & 1) * 8) * 2;
    const int j_end = CAUSAL ? i + 1 : n_t;
    for (int j = 0; j < j_end; ++j) {
      const int kv0 = j * 16;
      uint32_t dsa[4];
      ldsm_x4_t(dsa, ds_lane + kv0 * dstride);
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bb[4];
        load_b_kn(bb, uK, kv0, np * 16, lane);
        mma16816(dq[2 * np], dsa, bb[0], bb[1]);
        mma16816(dq[2 * np + 1], dsa, bb[2], bb[3]);
      }
    }
    const int r0 = q0 + g, r1 = r0 + 8;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      if (r0 < S) *reinterpret_cast<uint32_t*>(dbase + (long long)r0 * ld + nt * 8 + 2 * t) = pack_bf16x2(dq[nt][0], dq[nt][1]);
      if (r1 < S) *reinterpret_cast<uint32_t*>(dbase + (long long)r1 * ld + nt * 8 + 2 * t) = pack_bf16x2(dq[nt][2], dq[nt][3]);
    }
  }
}

// warps per CTA: at most 8, with the 16-row tiles spread evenly over them
static int pick_threads(int S) {
  const int n_t = (S + 15) / 16;
  const int per = (n_t + 7) / 8;
  return ((n_t + per - 1) / per) * 32;
}

static int attention_fwd_impl(const void* qkv, void* out, float* lse, const uint8_t* kmask, int B, int S, int H,
                              int causal, float scale, void* stream) {
  if (B <= 0 || S <= 0 || H <= 0) return MMB_ERR_UNSUPPORTED;
  if (S > SMAX)   // the head no longer fits in shared memory: stream K / V
    return attention_fwd_stream(qkv, out, lse, kmask, B, S, H, causal, scale, reinterpret_cast<cudaStream_t>(stream));
  const int S_pad = (S + 15) & ~15;
  const int smem = 3 * S_pad * 128 + 8 * (SMAX / 64) + S_pad;
  const float scale_log2 = scale * 1.4426950408889634f;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  auto kfn = causal ? attn_fwd_kernel<true> : attn_fwd_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return (int)e;
  kfn<<<B * H, pick_threads(S), smem, st>>>((const __nv_bfloat16*)qkv, (__nv_bfloat16*)out, lse, kmask, S, H, scale_log2);
  return (int)cudaGetLastError();
}

static int attention_bwd_impl(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                              const uint8_t* kmask, int B, int S, int H, int causal, float scale, void* stream) {
  if (B <= 0 || S <= 0 || H <= 0) return MMB_ERR_UNSUPPORTED;
  if (S > SMAX)
    return attention_bwd_stream(qkv, out, dout, lse, dqkv, kmask, B, S, H, causal, scale,
                                reinterpret_cast<cudaStream_t>(stream));
  const int S_pad = (S + 15) & ~15;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (S_pad <= BWD_STAGED_MAX) {   // Q, K, V, dO and dS^T fit in shared memory
    const int smem = bwd_staged_smem(S_pad);
    auto kfn = causal ? attn_bwd_staged_kernel<true> : attn_bwd_staged_kernel<false>;
    cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    kfn<<<B * H, (S_pad / 16) * 32, smem, st>>>((const __nv_bfloat16*)qkv, (const __nv_bfloat16*)out,
                                                (const __nv_bfloat16*)dout, lse, kmask, (__nv_bfloat16*)dqkv, S, H, scale);
    return (int)cudaGetLastError();
  }
  const int smem = 4 * S_pad * 128 + 2 * S_pad * 4 + S_pad;
  auto kfn = causal ? attn_bwd_kernel<true> : attn_bwd_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return (int)e;
  kfn<<<B * H, pick_threads(S), smem, st>>>((const __nv_bfloat16*)qkv, (const __nv_bfloat16*)out,
                                            (const __nv_bfloat16*)dout, lse, kmask, (__nv_bfloat16*)dqkv, S, H, scale);
  return (int)cudaGetLastError();
}

}  // namespace mmb

using namespace mmb;

// kernels one mmb_attention_bwd call launches at sequence length S (callers that count launches: bench.py)
extern "C" int mmb_attention_bwd_launches(int S) { return S > SMAX ? ATTN_BWD_STREAM_LAUNCHES : 1; }

extern "C" int mmb_attention_fwd(const void* qkv, void* out, float* lse, int B, int S, int H, int head_dim, int causal,
                                 float scale, void* stream) {
  if (head_dim != HD) return MMB_ERR_UNSUPPORTED;
  return attention_fwd_impl(qkv, out, lse, nullptr, B, S, H, causal, scale, stream);
}
// Same with a key-padding mask [B,S] (1 = attend): BERT-style attention of the FLAVA text tower
// (modules/encoders/bert_text_encoder.py:87-93 -> modules/layers/attention.py:228-229 masked_fill(-inf)).
extern "C" int mmb_attention_fwd_kmask(const void* qkv, void* out, float* lse, const unsigned char* kmask, int B, int S,
                                       int H, int head_dim, int causal, float scale, void* stream) {
  if (head_dim != HD) return MMB_ERR_UNSUPPORTED;
  return attention_fwd_impl(qkv, out, lse, kmask, B, S, H, causal, scale, stream);
}
extern "C" int mmb_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                                 int B, int S, int H, int head_dim, int causal, float scale, void* stream) {
  if (head_dim != HD) return MMB_ERR_UNSUPPORTED;
  return attention_bwd_impl(qkv, out, dout, lse, dqkv, nullptr, B, S, H, causal, scale, stream);
}
// Backward of mmb_attention_fwd_kmask: masked keys get P = dS = 0, i.e. zero dK / dV rows and no share in dQ
// (modules/layers/attention.py:220-239 under autograd, additive -inf mask of utils/attention.py:13-53).
extern "C" int mmb_attention_bwd_kmask(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                                       const unsigned char* kmask, int B, int S, int H, int head_dim, int causal,
                                       float scale, void* stream) {
  if (head_dim != HD) return MMB_ERR_UNSUPPORTED;
  return attention_bwd_impl(qkv, out, dout, lse, dqkv, kmask, B, S, H, causal, scale, stream);
}
