// Backward of the general attention forward (attention_generic.cu): cross-attention, head_dim 64 / 96 / 128,
// batch-shared (learned) queries, arbitrary boolean masks — the CoCa poolers, the text decoder's [causal x padding] mask
// and the multimodal decoder's cross-attention under autograd (modules/layers/multi_head_attention.py:74-76,171-173).
// These are ~3 % of CoCa's FLOPs, so this is a plain SIMT design chosen for being easy to verify, not a tensor-core one.
// Two generations live here: the row-per-warp kernels described first (fallback: MMB_ATTN_GEN_BWD=rows, and Skv > 512 for
// the query kernel) and their shared-memory tiled variants (default; 3.1x faster at CoCa ViT-L/14 shapes), further down.
//
//   kernel Q : one warp per (batch, head, query i), lane = key within blocks of 32.  Skv <= 512: one sweep, the lane's scores
//              and dP stay in registers (row LSE -> D_i = sum_j p_ij dP_ij -> dS_ij = p_ij (dP_ij - D_i) scale); longer key
//              sequences: three sweeps that recompute them.  dQ_i = sum_j dS_ij k_j is accumulated with lane = channel
//              group (dS broadcast by shuffle).  Writes LSE_i / D_i for kernel KV.
//   kernel KV: one warp per (batch, head, key j).  Sweeps the queries in blocks of 32 (lane = query), recomputes
//              p_ij / dS_ij from LSE_i / D_i and accumulates dV_j = sum_i p_ij dO_i, dK_j = sum_i dS_ij q_i.
//
// No atomics except for batch-shared queries (bsq == 0), whose gradient is the sum over the batch (fp32 atomics into
// dq_f32).  fp32 arithmetic throughout; p is NOT rounded to bf16 (the forward rounds P for its PV product; the
// difference is below the bf16 noise of the operands).  A fully masked query row has p = 0 everywhere (as the forward).
#include <cstdlib>

#include "attention_generic.cuh"
#include "mmb200_internal.h"

namespace mmb {

__device__ __forceinline__ float wred_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float wred_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float dot_row(const __nv_bfloat16* __restrict__ row, const float* __restrict__ vec, int hd) {
  float acc = 0.f;
  for (int c = 0; c < hd; c += 8) {   // rows are 16-byte aligned (strides are multiples of 8 elements)
    const uint4 u = *reinterpret_cast<const uint4*>(row + c);
    acc += bf16_lo(u.x) * vec[c] + bf16_hi(u.x) * vec[c + 1] + bf16_lo(u.y) * vec[c + 2] + bf16_hi(u.y) * vec[c + 3] +
           bf16_lo(u.z) * vec[c + 4] + bf16_hi(u.z) * vec[c + 5] + bf16_lo(u.w) * vec[c + 6] + bf16_hi(u.w) * vec[c + 7];
  }
  return acc;
}
__device__ __forceinline__ bool attends(const AttnGenBwdArgs& a, int b, int i, int j) {
  if (a.causal && j > i) return false;
  if (a.mask && !a.mask[b * a.mask_bs + i * a.mask_qs + j]) return false;
  return true;
}

template <int HD>
__global__ void __launch_bounds__(256) attn_gen_bwd_q_kernel(const AttnGenBwdArgs a) {
  constexpr int CPL = HD / 32;   // channels per lane in the accumulation phase
  __shared__ float sq[8][HD], sdo[8][HD];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + warp;
  const long long total = (long long)a.B * a.H * a.Sq;
  if (row >= total) return;   // whole warp
  const int i = (int)(row % a.Sq);
  const int h = (int)((row / a.Sq) % a.H);
  const int b = (int)(row / ((long long)a.Sq * a.H));
  const __nv_bfloat16* qrow = a.q + b * a.bsq + (long long)i * a.ldq + h * HD;
  const __nv_bfloat16* dorow = a.dout + b * a.bso + (long long)i * a.ldo + h * HD;
  const __nv_bfloat16* kbase = a.k + b * a.bsk + h * HD;
  const __nv_bfloat16* vbase = a.v + b * a.bsv + h * HD;
  float* q = sq[warp];
  float* dO = sdo[warp];
  for (int c = lane; c < HD; c += 32) { q[c] = __bfloat162float(qrow[c]); dO[c] = __bfloat162float(dorow[c]); }
  __syncwarp();
  float acc[CPL];
#pragma unroll
  for (int e = 0; e < CPL; ++e) acc[e] = 0.f;
  constexpr int KB = 16;   // key blocks whose scores / dP one lane keeps in registers: Skv <= 512
  if (a.Skv <= 32 * KB) {
    // ---- one sweep over the keys: s_j and dP_j of this lane's keys stay in registers (2 dot products per pair instead
    //      of the 5 of the three-sweep path below)
    const int nb = (a.Skv + 31) >> 5;
    float sc[KB], dp[KB];
    float mx = -INFINITY;
#pragma unroll
    for (int jb = 0; jb < KB; ++jb) {
      sc[jb] = -INFINITY;
      dp[jb] = 0.f;
      if (jb < nb) {
        const int j = jb * 32 + lane;
        if (j < a.Skv && attends(a, b, i, j)) {
          sc[jb] = dot_row(kbase + (long long)j * a.ldk, q, HD) * a.scale_log2;
          dp[jb] = dot_row(vbase + (long long)j * a.ldv, dO, HD);
          mx = fmaxf(mx, sc[jb]);
        }
      }
    }
    mx = wred_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int jb = 0; jb < KB; ++jb)
      if (jb < nb && sc[jb] > -INFINITY) sum += exp2f(sc[jb] - mx);
    sum = wred_sum(sum);
    const float lse2 = (sum > 0.f) ? mx + log2f(sum) : INFINITY;
    float D = 0.f;
#pragma unroll
    for (int jb = 0; jb < KB; ++jb)
      if (jb < nb) {
        sc[jb] = (sc[jb] > -INFINITY) ? exp2f(sc[jb] - lse2) : 0.f;   // now p_j
        D += sc[jb] * dp[jb];
      }
    D = wred_sum(D);
    if (lane == 0) { a.lse[row] = lse2; a.dsum[row] = D; }
#pragma unroll
    for (int jb = 0; jb < KB; ++jb)
      if (jb < nb) {
        const float ds = sc[jb] * (dp[jb] - D) * a.scale;
        const int j0 = jb * 32, nj = min(32, a.Skv - j0);
        for (int t = 0; t < nj; ++t) {
          const float dst = __shfl_sync(0xffffffffu, ds, t);
          if (dst != 0.f) {   // uniform across the warp
            const __nv_bfloat16* kr = kbase + (long long)(j0 + t) * a.ldk + lane * CPL;
#pragma unroll
            for (int e = 0; e < CPL; ++e) acc[e] += dst * __bfloat162float(kr[e]);
          }
        }
      }
  } else {
  // ---- three-sweep path (any Skv): sweep 1: row max / sum (log2 domain)
  float mx = -INFINITY;
  for (int j0 = 0; j0 < a.Skv; j0 += 32) {
    const int j = j0 + lane;
    if (j < a.Skv && attends(a, b, i, j)) mx = fmaxf(mx, dot_row(kbase + (long long)j * a.ldk, q, HD) * a.scale_log2);
  }
  mx = wred_max(mx);
  float sum = 0.f;
  if (mx > -INFINITY) {
    for (int j0 = 0; j0 < a.Skv; j0 += 32) {
      const int j = j0 + lane;
      if (j < a.Skv && attends(a, b, i, j)) sum += exp2f(dot_row(kbase + (long long)j * a.ldk, q, HD) * a.scale_log2 - mx);
    }
  }
  sum = wred_sum(sum);
  const float lse2 = (sum > 0.f) ? mx + log2f(sum) : INFINITY;   // fully masked row: p = exp2(s - inf) = 0
  // sweep 2: D = sum_j p_j dP_j
  float D = 0.f;
  for (int j0 = 0; j0 < a.Skv; j0 += 32) {
    const int j = j0 + lane;
    if (j < a.Skv && attends(a, b, i, j)) {
      const float p = exp2f(dot_row(kbase + (long long)j * a.ldk, q, HD) * a.scale_log2 - lse2);
      D += p * dot_row(vbase + (long long)j * a.ldv, dO, HD);
    }
  }
  D = wred_sum(D);
  if (lane == 0) { a.lse[row] = lse2; a.dsum[row] = D; }
  // sweep 3: dS and dQ
  for (int j0 = 0; j0 < a.Skv; j0 += 32) {
    const int j = j0 + lane;
    float ds = 0.f;
    if (j < a.Skv && attends(a, b, i, j)) {
      const float p = exp2f(dot_row(kbase + (long long)j * a.ldk, q, HD) * a.scale_log2 - lse2);
      ds = p * (dot_row(vbase + (long long)j * a.ldv, dO, HD) - D) * a.scale;
    }
    const int nj = min(32, a.Skv - j0);
    for (int t = 0; t < nj; ++t) {
      const float dst = __shfl_sync(0xffffffffu, ds, t);
      if (dst != 0.f) {   // uniform across the warp
        const __nv_bfloat16* kr = kbase + (long long)(j0 + t) * a.ldk + lane * CPL;
#pragma unroll
        for (int e = 0; e < CPL; ++e) acc[e] += dst * __bfloat162float(kr[e]);
      }
    }
  }
  }   // three-sweep path
  if (a.dq) {
    __nv_bfloat16* o = a.dq + b * a.bsq + (long long)i * a.ldq + h * HD + lane * CPL;
#pragma unroll
    for (int e = 0; e < CPL; ++e) o[e] = __float2bfloat16(acc[e]);
  }
  if (a.dq_f32) {
    float* o = a.dq_f32 + (long long)i * a.ldq32 + h * HD + lane * CPL;
#pragma unroll
    for (int e = 0; e < CPL; ++e) atomicAdd(o + e, acc[e]);
  }
}

template <int HD>
__global__ void __launch_bounds__(256) attn_gen_bwd_kv_kernel(const AttnGenBwdArgs a) {
  constexpr int CPL = HD / 32;
  __shared__ float sk[8][HD], sv[8][HD];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + warp;
  const long long total = (long long)a.B * a.H * a.Skv;
  if (row >= total) return;
  const int j = (int)(row % a.Skv);
  const int h = (int)((row / a.Skv) % a.H);
  const int b = (int)(row / ((long long)a.Skv * a.H));
  const __nv_bfloat16* krow = a.k + b * a.bsk + (long long)j * a.ldk + h * HD;
  const __nv_bfloat16* vrow = a.v + b * a.bsv + (long long)j * a.ldv + h * HD;
  const __nv_bfloat16* qbase = a.q + b * a.bsq + h * HD;
  const __nv_bfloat16* dobase = a.dout + b * a.bso + h * HD;
  const float* lse = a.lse + ((long long)b * a.H + h) * a.Sq;
  const float* dsum = a.dsum + ((long long)b * a.H + h) * a.Sq;
  float* kf = sk[warp];
  float* vf = sv[warp];
  for (int c = lane; c < HD; c += 32) { kf[c] = __bfloat162float(krow[c]); vf[c] = __bfloat162float(vrow[c]); }
  __syncwarp();
  float accK[CPL], accV[CPL];
#pragma unroll
  for (int e = 0; e < CPL; ++e) { accK[e] = 0.f; accV[e] = 0.f; }
  for (int i0 = 0; i0 < a.Sq; i0 += 32) {
    const int i = i0 + lane;
    float p = 0.f, ds = 0.f;
    if (i < a.Sq && attends(a, b, i, j)) {
      p = exp2f(dot_row(qbase + (long long)i * a.ldq, kf, HD) * a.scale_log2 - lse[i]);
      ds = p * (dot_row(dobase + (long long)i * a.ldo, vf, HD) - dsum[i]) * a.scale;
    }
    const int ni = min(32, a.Sq - i0);
    for (int t = 0; t < ni; ++t) {
      const float pt = __shfl_sync(0xffffffffu, p, t);
      const float dst = __shfl_sync(0xffffffffu, ds, t);
      if (pt != 0.f) {   // uniform across the warp (ds is 0 whenever p is)
        const __nv_bfloat16* qr = qbase + (long long)(i0 + t) * a.ldq + lane * CPL;
        const __nv_bfloat16* dr = dobase + (long long)(i0 + t) * a.ldo + lane * CPL;
#pragma unroll
        for (int e = 0; e < CPL; ++e) {
          accV[e] += pt * __bfloat162float(dr[e]);
          accK[e] += dst * __bfloat162float(qr[e]);
        }
      }
    }
  }
  __nv_bfloat16* ok = a.dk + b * a.bsk + (long long)j * a.ldk + h * HD + lane * CPL;
  __nv_bfloat16* ov = a.dv + b * a.bsv + (long long)j * a.ldv + h * HD + lane * CPL;
#pragma unroll
  for (int e = 0; e < CPL; ++e) { ok[e] = __float2bfloat16(accK[e]); ov[e] = __float2bfloat16(accV[e]); }
}

// ---------------------------------------------------------------------------------------------------------------------
// Tiled variants (the default): the 8 warps of a CTA work on 8 consecutive rows of ONE (batch, head), and the 32-row blocks
// of the other sequence are staged in shared memory once per CTA (coalesced 16-byte loads) instead of being read row by
// row, per lane, from global memory by every warp.  Row pitch HD*2 + 16 bytes: an odd number of 16-byte chunks, so the 32
// lanes' row reads are bank-conflict-free.  Same arithmetic, in the same order, as the kernels above.
// ---------------------------------------------------------------------------------------------------------------------
template <int HD>
__device__ __forceinline__ float dot_smem(const __nv_bfloat16* __restrict__ row, const float* __restrict__ vec) {
  float acc = 0.f;
#pragma unroll
  for (int c = 0; c < HD; c += 8) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + c);
    acc += bf16_lo(u.x) * vec[c] + bf16_hi(u.x) * vec[c + 1] + bf16_lo(u.y) * vec[c + 2] + bf16_hi(u.y) * vec[c + 3] +
           bf16_lo(u.z) * vec[c + 4] + bf16_hi(u.z) * vec[c + 5] + bf16_lo(u.w) * vec[c + 6] + bf16_hi(u.w) * vec[c + 7];
  }
  return acc;
}

// rows [r0, r0 + 32) of a [n_rows, HD] bf16 matrix (row stride ld) -> tile[32][HD + 8]; rows past n_rows are zero-filled
template <int HD>
__device__ __forceinline__ void load_tile32(__nv_bfloat16* __restrict__ tile, const __nv_bfloat16* __restrict__ base,
                                            long long ld, int r0, int n_rows) {
  constexpr int C8 = HD / 8;
  for (int idx = threadIdx.x; idx < 32 * C8; idx += blockDim.x) {
    const int r = idx / C8, c = (idx % C8) * 8;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r0 + r < n_rows) v = *reinterpret_cast<const uint4*>(base + (long long)(r0 + r) * ld + c);
    *reinterpret_cast<uint4*>(tile + r * (HD + 8) + c) = v;
  }
}

template <int HD>
__global__ void __launch_bounds__(256) attn_gen_bwd_q_tiled_kernel(const AttnGenBwdArgs a) {
  constexpr int CPL = HD / 32, KB = 16, PITCH = HD + 8;
  __shared__ __align__(16) __nv_bfloat16 sK[32 * PITCH];
  __shared__ __align__(16) __nv_bfloat16 sV[32 * PITCH];
  __shared__ float sq[8][HD], sdo[8][HD];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * 8 + warp, h = blockIdx.y, b = blockIdx.z;
  const bool valid = i < a.Sq;
  const __nv_bfloat16* kbase = a.k + b * a.bsk + h * HD;
  const __nv_bfloat16* vbase = a.v + b * a.bsv + h * HD;
  float* q = sq[warp];
  float* dO = sdo[warp];
  if (valid) {
    const __nv_bfloat16* qrow = a.q + b * a.bsq + (long long)i * a.ldq + h * HD;
    const __nv_bfloat16* dorow = a.dout + b * a.bso + (long long)i * a.ldo + h * HD;
    for (int c = lane; c < HD; c += 32) { q[c] = __bfloat162float(qrow[c]); dO[c] = __bfloat162float(dorow[c]); }
  }
  const int nb = (a.Skv + 31) >> 5;   // <= KB (checked by the launcher)
  float sc[KB], dp[KB];
  float mx = -INFINITY;
#pragma unroll
  for (int jb = 0; jb < KB; ++jb) {
    sc[jb] = -INFINITY;
    dp[jb] = 0.f;
    if (jb < nb) {                     // uniform over the CTA
      __syncthreads();                 // the previous block's tile reads (and the q / dO staging) are done
      load_tile32<HD>(sK, kbase, a.ldk, jb * 32, a.Skv);
      load_tile32<HD>(sV, vbase, a.ldv, jb * 32, a.Skv);
      __syncthreads();
      const int j = jb * 32 + lane;
      if (valid && j < a.Skv && attends(a, b, i, j)) {
        sc[jb] = dot_smem<HD>(sK + lane * PITCH, q) * a.scale_log2;
        dp[jb] = dot_smem<HD>(sV + lane * PITCH, dO);
        mx = fmaxf(mx, sc[jb]);
      }
    }
  }
  if (!valid) return;                  // no block-wide synchronisation below
  mx = wred_max(mx);
  float sum = 0.f;
#pragma unroll
  for (int jb = 0; jb < KB; ++jb)
    if (jb < nb && sc[jb] > -INFINITY) sum += exp2f(sc[jb] - mx);
  sum = wred_sum(sum);
  const float lse2 = (sum > 0.f) ? mx + log2f(sum) : INFINITY;
  float D = 0.f;
#pragma unroll
  for (int jb = 0; jb < KB; ++jb)
    if (jb < nb) {
      sc[jb] = (sc[jb] > -INFINITY) ? exp2f(sc[jb] - lse2) : 0.f;   // now p_j
      D += sc[jb] * dp[jb];
    }
  D = wred_sum(D);
  const long long row = ((long long)b * a.H + h) * a.Sq + i;
  if (lane == 0) { a.lse[row] = lse2; a.dsum[row] = D; }
  float acc[CPL];
#pragma unroll
  for (int e = 0; e < CPL; ++e) acc[e] = 0.f;
#pragma unroll
  for (int jb = 0; jb < KB; ++jb)
    if (jb < nb) {
      const float ds = sc[jb] * (dp[jb] - D) * a.scale;
      const int j0 = jb * 32, nj = min(32, a.Skv - j0);
      for (int t = 0; t < nj; ++t) {
        const float dst = __shfl_sync(0xffffffffu, ds, t);
        if (dst != 0.f) {   // uniform across the warp
          const __nv_bfloat16* kr = kbase + (long long)(j0 + t) * a.ldk + lane * CPL;
#pragma unroll
          for (int e = 0; e < CPL; ++e) acc[e] += dst * __bfloat162float(kr[e]);
        }
      }
    }
  if (a.dq) {
    __nv_bfloat16* o = a.dq + b * a.bsq + (long long)i * a.ldq + h * HD + lane * CPL;
#pragma unroll
    for (int e = 0; e < CPL; ++e) o[e] = __float2bfloat16(acc[e]);
  }
  if (a.dq_f32) {
    float* o = a.dq_f32 + (long long)i * a.ldq32 + h * HD + lane * CPL;
#pragma unroll
    for (int e = 0; e < CPL; ++e) atomicAdd(o + e, acc[e]);
  }
}

template <int HD>
__global__ void __launch_bounds__(256) attn_gen_bwd_kv_tiled_kernel(const AttnGenBwdArgs a) {
  constexpr int CPL = HD / 32, PITCH = HD + 8;
  __shared__ __align__(16) __nv_bfloat16 sQ[32 * PITCH];
  __shared__ __align__(16) __nv_bfloat16 sDO[32 * PITCH];
  __shared__ float sk[8][HD], sv[8][HD];
  __shared__ float sL[32], sD[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = blockIdx.x * 8 + warp, h = blockIdx.y, b = blockIdx.z;
  const bool valid = j < a.Skv;
  const __nv_bfloat16* qbase = a.q + b * a.bsq + h * HD;
  const __nv_bfloat16* dobase = a.dout + b * a.bso + h * HD;
  const float* lse = a.lse + ((long long)b * a.H + h) * a.Sq;
  const float* dsum = a.dsum + ((long long)b * a.H + h) * a.Sq;
  float* kf = sk[warp];
  float* vf = sv[warp];
  if (valid) {
    const __nv_bfloat16* krow = a.k + b * a.bsk + (long long)j * a.ldk + h * HD;
    const __nv_bfloat16* vrow = a.v + b * a.bsv + (long long)j * a.ldv + h * HD;
    for (int c = lane; c < HD; c += 32) { kf[c] = __bfloat162float(krow[c]); vf[c] = __bfloat162float(vrow[c]); }
  }
  float accK[CPL], accV[CPL];
#pragma unroll
  for (int e = 0; e < CPL; ++e) { accK[e] = 0.f; accV[e] = 0.f; }
  for (int i0 = 0; i0 < a.Sq; i0 += 32) {   // uniform over the CTA
    __syncthreads();
    load_tile32<HD>(sQ, qbase, a.ldq, i0, a.Sq);
    load_tile32<HD>(sDO, dobase, a.ldo, i0, a.Sq);
    if (threadIdx.x < 32) {
      const int i = i0 + threadIdx.x;
      sL[threadIdx.x] = i < a.Sq ? lse[i] : INFINITY;
      sD[threadIdx.x] = i < a.Sq ? dsum[i] : 0.f;
    }
    __syncthreads();
    if (valid) {
      const int i = i0 + lane;
      float p = 0.f, ds = 0.f;
      if (i < a.Sq && attends(a, b, i, j)) {
        p = exp2f(dot_smem<HD>(sQ + lane * PITCH, kf) * a.scale_log2 - sL[lane]);
        ds = p * (dot_smem<HD>(sDO + lane * PITCH, vf) - sD[lane]) * a.scale;
      }
      const int ni = min(32, a.Sq - i0);
      for (int t = 0; t < ni; ++t) {
        const float pt = __shfl_sync(0xffffffffu, p, t);
        const float dst = __shfl_sync(0xffffffffu, ds, t);
        if (pt != 0.f) {   // uniform across the warp (ds is 0 whenever p is)
          const __nv_bfloat16* qr = sQ + t * PITCH + lane * CPL;
          const __nv_bfloat16* dr = sDO + t * PITCH + lane * CPL;
#pragma unroll
          for (int e = 0; e < CPL; ++e) {
            accV[e] += pt * __bfloat162float(dr[e]);
            accK[e] += dst * __bfloat162float(qr[e]);
          }
        }
      }
    }
  }
  if (!valid) return;
  __nv_bfloat16* ok = a.dk + b * a.bsk + (long long)j * a.ldk + h * HD + lane * CPL;
  __nv_bfloat16* ov = a.dv + b * a.bsv + (long long)j * a.ldv + h * HD + lane * CPL;
#pragma unroll
  for (int e = 0; e < CPL; ++e) { ok[e] = __float2bfloat16(accK[e]); ov[e] = __float2bfloat16(accV[e]); }
}

template <int HD>
static int launch_gen_bwd(const AttnGenBwdArgs& a, cudaStream_t st) {
  const long long nq = (long long)a.B * a.H * a.Sq, nk = (long long)a.B * a.H * a.Skv;
  static int tiled = -1;   // MMB_ATTN_GEN_BWD=rows selects the row-per-warp kernels (A/B, fallback)
  if (tiled < 0) {
    const char* e = getenv("MMB_ATTN_GEN_BWD");
    tiled = (e && e[0] == 'r') ? 0 : 1;
  }
  const bool grid_ok = a.H <= 65535 && a.B <= 65535;
  if (tiled && grid_ok && a.Skv <= 512)
    attn_gen_bwd_q_tiled_kernel<HD><<<dim3((a.Sq + 7) / 8, a.H, a.B), 256, 0, st>>>(a);
  else
    attn_gen_bwd_q_kernel<HD><<<(unsigned)((nq + 7) / 8), 256, 0, st>>>(a);
  if (tiled && grid_ok)
    attn_gen_bwd_kv_tiled_kernel<HD><<<dim3((a.Skv + 7) / 8, a.H, a.B), 256, 0, st>>>(a);
  else
    attn_gen_bwd_kv_kernel<HD><<<(unsigned)((nk + 7) / 8), 256, 0, st>>>(a);
  return (int)cudaGetLastError();
}

}  // namespace mmb

using namespace mmb;

// dq / dk / dv share the strides of q / k / v.  dq_bf16 may be NULL; dq_f32 (optional, [Sq, ldq32] fp32, accumulated with
// atomics — zero it first) is the gradient of batch-shared queries (bsq = 0), summed over the batch.
// scratch: fp32 [2 * B * H * Sq] (row LSE and D), written by the query kernel and read by the key/value kernel.
extern "C" int mmb_attention_bwd_generic(const void* q, long long ldq, long long bsq, const void* k, long long ldk,
                                         long long bsk, const void* v, long long ldv, long long bsv, const void* dout,
                                         long long ldo, long long bso, const void* mask, long long mask_bs,
                                         long long mask_qs, void* dq_bf16, float* dq_f32, long long ldq32, void* dk_bf16,
                                         void* dv_bf16, float* scratch, int B, int Sq, int Skv, int H, int head_dim,
                                         int causal, float scale, void* stream) {
  if (B <= 0 || Sq <= 0 || Skv <= 0 || H <= 0 || !scratch || !dk_bf16 || !dv_bf16) return MMB_ERR_ARG;
  if ((ldq | ldk | ldv | ldo | bsq | bsk | bsv | bso) & 7) return MMB_ERR_ARG;   // 16-byte row loads
  if ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
       reinterpret_cast<uintptr_t>(dout)) & 15)
    return MMB_ERR_ARG;
  if (bsq == 0 && B > 1 && dq_bf16 != nullptr) return MMB_ERR_ARG;              // shared queries: use dq_f32 (summed over b)
  AttnGenBwdArgs a{};
  a.q = (const __nv_bfloat16*)q; a.k = (const __nv_bfloat16*)k; a.v = (const __nv_bfloat16*)v;
  a.dout = (const __nv_bfloat16*)dout;
  a.ldq = ldq; a.ldk = ldk; a.ldv = ldv; a.ldo = ldo; a.bsq = bsq; a.bsk = bsk; a.bsv = bsv; a.bso = bso;
  a.mask = (const uint8_t*)mask; a.mask_bs = mask_bs; a.mask_qs = mask_qs;
  a.dq = (__nv_bfloat16*)dq_bf16; a.dk = (__nv_bfloat16*)dk_bf16; a.dv = (__nv_bfloat16*)dv_bf16;
  a.dq_f32 = dq_f32; a.ldq32 = ldq32;
  a.lse = scratch; a.dsum = scratch + (long long)B * H * Sq;
  a.B = B; a.Sq = Sq; a.Skv = Skv; a.H = H; a.causal = causal;
  a.scale = scale; a.scale_log2 = scale * 1.4426950408889634f;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (head_dim != 64 && head_dim != 96 && head_dim != 128) return MMB_ERR_UNSUPPORTED;
  // the shapes the resident forward serves keep the SIMT kernels; every longer one runs the streamed backward
  if (!generic_resident_fits(Sq, Skv, head_dim)) return attention_bwd_gstream(a, head_dim, st);
  switch (head_dim) {
    case 64: return launch_gen_bwd<64>(a, st);
    case 96: return launch_gen_bwd<96>(a, st);
    default: return launch_gen_bwd<128>(a, st);
  }
}
