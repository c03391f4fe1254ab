// HBM-bound backward kernels of the FLAVA / CoCa encoders' embedding, token-assembly, pooler and head stages
// (the forward counterparts live in elementwise.cu).  Same conventions: 128-bit coalesced accesses, one warp per token
// for the row-wise LayerNorm work, fp32 `red.global.add` for the scatter-adds into embedding tables.
#include "common.cuh"
#include "mmb200_internal.h"

namespace mmb {

__device__ __forceinline__ void red4(float* dst, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
static inline int grid_cap(long long n_items, int per_block) {
  long long b = (n_items + per_block - 1) / per_block;
  const long long cap = (long long)num_sms() * 16;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

constexpr int NVMAX = 8;   // d = 128 * nv, nv <= 8 (same bound as the forward LayerNorm kernels)

// Backward of bert_embed_ln_fwd_kernel: x = LN(word[ids] + pos[s] + type[tt]) * gamma + beta.
// Per token (one warp): the pre-LayerNorm sum and its statistics are RECOMPUTED from the tables (the forward keeps
// nothing), dx = rstd * (dy*gamma - mean(dy*gamma) - xhat * mean(dy*gamma*xhat)) is scatter-added into the three
// tables; dgamma / dbeta are accumulated per warp in registers over its tokens and flushed once.
// (autograd of modules/layers/text_embedding.py:70-104)
__global__ void __launch_bounds__(256) bert_embed_ln_bwd_kernel(
    const long long* __restrict__ ids, const long long* __restrict__ type_ids, const float* __restrict__ word,
    const float* __restrict__ pos, const float* __restrict__ type, const float* __restrict__ gamma,
    const float* __restrict__ dy, float* __restrict__ dword, float* __restrict__ dpos, float* __restrict__ dtype,
    float* __restrict__ dgamma, float* __restrict__ dbeta, int B, int S, int d, int V, float eps) {
  const int nv = d >> 7;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int M = B * S;
  float4 ag[NVMAX], ab[NVMAX];
#pragma unroll
  for (int i = 0; i < NVMAX; ++i) { ag[i] = make_float4(0.f, 0.f, 0.f, 0.f); ab[i] = ag[i]; }
  for (int m = blockIdx.x * wpb + (threadIdx.x >> 5); m < M; m += gridDim.x * wpb) {
    const int s = m % S;
    const long long tok = ids[m];
    if (tok < 0 || tok >= V) __trap();
    const long long ty = type_ids ? type_ids[m] : 0;
    float4 e[NVMAX];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < NVMAX; ++i)
      if (i < nv) {
        const int c = (i * 32 + lane) * 4;
        const float4 a = __ldg(reinterpret_cast<const float4*>(word + tok * d + c));
        const float4 b = __ldg(reinterpret_cast<const float4*>(pos + (long long)s * d + c));
        const float4 t = __ldg(reinterpret_cast<const float4*>(type + ty * d + c));
        e[i] = make_float4(a.x + b.x + t.x, a.y + b.y + t.y, a.z + b.z + t.z, a.w + b.w + t.w);
        sum += e[i].x + e[i].y + e[i].z + e[i].w;
      }
    const float mean = wsum(sum) / d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NVMAX; ++i)
      if (i < nv) {
        e[i].x -= mean; e[i].y -= mean; e[i].z -= mean; e[i].w -= mean;
        q += e[i].x * e[i].x + e[i].y * e[i].y + e[i].z * e[i].z + e[i].w * e[i].w;
      }
    const float rstd = rsqrtf(wsum(q) / d + eps);
    float4 g[NVMAX];   // dy * gamma
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NVMAX; ++i)
      if (i < nv) {
        const int c = (i * 32 + lane) * 4;
        const float4 y = *reinterpret_cast<const float4*>(dy + (long long)m * d + c);
        const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma + c));
        e[i].x *= rstd; e[i].y *= rstd; e[i].z *= rstd; e[i].w *= rstd;   // xhat
        ag[i].x += y.x * e[i].x; ag[i].y += y.y * e[i].y; ag[i].z += y.z * e[i].z; ag[i].w += y.w * e[i].w;
        ab[i].x += y.x; ab[i].y += y.y; ab[i].z += y.z; ab[i].w += y.w;
        g[i] = make_float4(y.x * gm.x, y.y * gm.y, y.z * gm.z, y.w * gm.w);
        s1 += g[i].x + g[i].y + g[i].z + g[i].w;
        s2 += g[i].x * e[i].x + g[i].y * e[i].y + g[i].z * e[i].z + g[i].w * e[i].w;
      }
    s1 = wsum(s1) / d;
    s2 = wsum(s2) / d;
#pragma unroll
    for (int i = 0; i < NVMAX; ++i)
      if (i < nv) {
        const int c = (i * 32 + lane) * 4;
        const float dx0 = rstd * (g[i].x - s1 - e[i].x * s2), dx1 = rstd * (g[i].y - s1 - e[i].y * s2);
        const float dx2 = rstd * (g[i].z - s1 - e[i].z * s2), dx3 = rstd * (g[i].w - s1 - e[i].w * s2);
        if (dword) red4(dword + tok * d + c, dx0, dx1, dx2, dx3);
        if (dpos) red4(dpos + (long long)s * d + c, dx0, dx1, dx2, dx3);
        if (dtype) red4(dtype + ty * d + c, dx0, dx1, dx2, dx3);
      }
  }
#pragma unroll
  for (int i = 0; i < NVMAX; ++i)
    if (i < nv) {
      const int c = (i * 32 + lane) * 4;
      if (dgamma) red4(dgamma + c, ag[i].x, ag[i].y, ag[i].z, ag[i].w);
      if (dbeta) red4(dbeta + c, ab[i].x, ab[i].y, ab[i].z, ab[i].w);
    }
}

// Backward of vit_assemble_fwd_kernel for the patch rows: dpatch[b*P+p] = bf16(mask[b,p] ? 0 : g[b,off+p]) and
// dmask_token += sum over masked (b,p) of g[b,off+p].  (dcls / dpos are batch sums of g: mmb_batch_sum.)
// One thread = one float4 column x a strip of ROWS consecutive patch rows (coalesced across the 4-column groups).
__global__ void __launch_bounds__(256) vit_assemble_bwd_kernel(const float* __restrict__ g,
                                                              const unsigned char* __restrict__ patch_mask,
                                                              __nv_bfloat16* __restrict__ dpatch,
                                                              float* __restrict__ dmask_token, int B, int S, int d,
                                                              int off, int rows_per_strip) {
  const int d4 = d >> 2;
  const int P = S - off;
  const long long n_rows = (long long)B * P;
  const long long n_strips = (n_rows + rows_per_strip - 1) / rows_per_strip;
  const long long total = n_strips * d4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d4) * 4;
    const long long r0 = (i / d4) * rows_per_strip;
    const long long r1 = r0 + rows_per_strip < n_rows ? r0 + rows_per_strip : n_rows;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long r = r0; r < r1; ++r) {
      const long long b = r / P;
      const int p = (int)(r % P);
      const float4 v = *reinterpret_cast<const float4*>(g + (b * S + off + p) * d + c);
      const bool masked = patch_mask != nullptr && patch_mask[r] != 0;
      uint2 o = make_uint2(0u, 0u);
      if (masked) { acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; }
      else { o.x = pack_bf16x2(v.x, v.y); o.y = pack_bf16x2(v.z, v.w); }
      *reinterpret_cast<uint2*>(dpatch + r * d + c) = o;
    }
    if (dmask_token != nullptr && patch_mask != nullptr) red4(dmask_token + c, acc.x, acc.y, acc.z, acc.w);
  }
}

// Inverse of concat_tokens_kernel for gradients: g [B, (cls?1:0)+Sa+Sb, d] fp32 -> a_bf16 [B*Sa, d], b_bf16 [B*Sb, d]
// (either may be NULL).  The cls row is left to mmb_batch_sum.
__global__ void split_tokens_cast_kernel(const float* __restrict__ g, __nv_bfloat16* __restrict__ a,
                                         __nv_bfloat16* __restrict__ bdst, int B, int Sa, int Sb, int d, int off) {
  const int d4 = d >> 2;
  const int So = off + Sa + Sb;
  const long long total = (long long)B * (Sa + Sb) * d4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d4) * 4;
    const long long row = i / d4;
    const int s = (int)(row % (Sa + Sb));
    const long long b = row / (Sa + Sb);
    const float4 v = *reinterpret_cast<const float4*>(g + (b * So + off + s) * d + c);
    uint2 o;
    o.x = pack_bf16x2(v.x, v.y);
    o.y = pack_bf16x2(v.z, v.w);
    if (s < Sa) { if (a) *reinterpret_cast<uint2*>(a + (b * Sa + s) * d + c) = o; }
    else        { if (bdst) *reinterpret_cast<uint2*>(bdst + (b * Sb + (s - Sa)) * d + c) = o; }
  }
}

// dx = dy * (1 - y^2)  (y = tanh(x));  outputs fp32 and / or bf16
__global__ void tanh_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dx,
                                __nv_bfloat16* __restrict__ dx_bf16, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float t = y[i];
    const float v = dy[i] * (1.f - t * t);
    if (dx) dx[i] = v;
    if (dx_bf16) dx_bf16[i] = __float2bfloat16(v);
  }
}

// dst[(b*rows_per_group + row), :] += src[b, :]   (gradient of "take token `row` of every sequence")
__global__ void scatter_rows_add_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int rows_per_group,
                                        int row, int d) {
  const int d4 = d >> 2;
  const long long total = (long long)B * d4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d4);
    const long long b = i / d4;
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    float4* p = reinterpret_cast<float4*>(dst + (b * rows_per_group + row) * d) + c;
    float4 o = *p;
    o.x += v.x; o.y += v.y; o.z += v.z; o.w += v.w;
    *p = o;
  }
}

// dst[idx[m], :] += src[m, :] for m < n (fp32; idx may repeat -> atomics): gradient of mmb_gather_rows_idx_cast
__global__ void scatter_rows_idx_add_kernel(const float* __restrict__ src, const long long* __restrict__ idx,
                                            float* __restrict__ dst, long long ld, int n, int d) {
  const int d4 = d >> 2;
  const long long total = (long long)n * d4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d4) * 4;
    const long long m = i / d4;
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    red4(dst + idx[m] * ld + c, v.x, v.y, v.z, v.w);
  }
}

// Cross-entropy backward on materialised fp32 logits (label-indexed, ignore_index; mean over kept rows):
//   dlogits[m, v] = bf16( w * (exp(logits[m,v] - lse[m]) - [v == label[m]]) ),  w = grad_scale / max(count, 1) for kept
//   rows and 0 for ignored rows (grad_scale: host factor x optional device scalar).  lse is recomputed per row here (one CTA per row: max pass, sum pass, write pass).
// (autograd of F.cross_entropy(ignore_index) in modules/losses/flava.py:143-238 and models/coca/coca_model.py:443-454)
__global__ void __launch_bounds__(256) ce_labels_bwd_kernel(const float* __restrict__ logits, long long ld,
                                                           const long long* __restrict__ labels, long long label_stride,
                                                           long long ignore_index, int V, const float* __restrict__ accum,
                                                           float grad_scale, const float* __restrict__ gscale_dev,
                                                           __nv_bfloat16* __restrict__ dlogits, long long ldd) {
  __shared__ float red[8];
  __shared__ float bc;
  const int m = blockIdx.x;
  const long long lab = labels[(long long)m * label_stride];
  const float* row = logits + (long long)m * ld;
  __nv_bfloat16* out = dlogits + (long long)m * ldd;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lab == ignore_index) {
    for (int v = threadIdx.x; v < V; v += blockDim.x) out[v] = __float2bfloat16(0.f);
    return;
  }
  if (lab < 0 || lab >= V) __trap();
  float mx = -INFINITY;
  for (int v = threadIdx.x; v < V; v += blockDim.x) mx = fmaxf(mx, row[v]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = red[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) t = fmaxf(t, red[i]);
    bc = t;
  }
  __syncthreads();
  mx = bc;
  float s = 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) s += __expf(row[v] - mx);
  s = wsum(s);
  __syncthreads();
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
    bc = t;
  }
  __syncthreads();
  const float inv = 1.f / bc;
  const float cnt = accum ? fmaxf(accum[1], 1.f) : 1.f;
  const float w = grad_scale * (gscale_dev ? gscale_dev[0] : 1.f) / cnt;   // gscale_dev: the incoming d loss, on the device
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    const float pv = __expf(row[v] - mx) * inv;
    out[v] = __float2bfloat16(w * (pv - (v == lab ? 1.f : 0.f)));
  }
}

// dx = bf16(dy * act'(pre)) on bf16 tensors: the activation backward when the gradient does not come out of a GEMM
// epilogue (EPI_BF16_DACT covers that case) — MaskedPredictionHead: LayerNorm backward -> GELU' (losses/flava.py:174-180)
template <int ACT>
__global__ void act_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ pre,
                               __nv_bfloat16* __restrict__ dx, long long n) {
  const long long n2 = n >> 1;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n2; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t a = reinterpret_cast<const uint32_t*>(dy)[i], b = reinterpret_cast<const uint32_t*>(pre)[i];
    reinterpret_cast<uint32_t*>(dx)[i] = pack_bf16x2(act_dgrad<ACT>(bf16_lo(a), bf16_lo(b)), act_dgrad<ACT>(bf16_hi(a), bf16_hi(b)));
  }
  if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0)
    dx[n - 1] = __float2bfloat16(act_dgrad<ACT>(__bfloat162float(dy[n - 1]), __bfloat162float(pre[n - 1])));
}

}  // namespace mmb

using namespace mmb;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define LAUNCH_RC() ((int)cudaGetLastError())

extern "C" int mmb_bert_embed_ln_bwd(const long long* ids, const long long* type_ids, const float* word, const float* pos,
                                     const float* type, const float* gamma, const float* dy, float* dword, float* dpos,
                                     float* dtype, float* dgamma, float* dbeta, int B, int S, int d, int V, float eps,
                                     void* stream) {
  if (d <= 0 || (d & 127) || (d >> 7) > NVMAX) return MMB_ERR_UNSUPPORTED;
  if (B <= 0 || S <= 0) return MMB_ERR_ARG;
  // few, long-lived warps: every warp flushes its dgamma / dbeta partial sums once (2 * d atomics per warp)
  long long blocks = ((long long)B * S + 8 * 16 - 1) / (8 * 16);
  const long long cap = (long long)num_sms() * 2;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  bert_embed_ln_bwd_kernel<<<(int)blocks, 256, 0, ST(stream)>>>(ids, type_ids, word, pos, type, gamma, dy, dword, dpos,
                                                                dtype, dgamma, dbeta, B, S, d, V, eps);
  return LAUNCH_RC();
}

extern "C" int mmb_vit_assemble_bwd(const float* g, const unsigned char* patch_mask, void* dpatch_bf16,
                                    float* dmask_token, int B, int S, int d, int has_cls, void* stream) {
  if ((d & 3) || B <= 0 || S <= (has_cls ? 1 : 0)) return MMB_ERR_ARG;
  const int rows_per_strip = 16;
  const long long strips = ((long long)B * (S - (has_cls ? 1 : 0)) + rows_per_strip - 1) / rows_per_strip;
  vit_assemble_bwd_kernel<<<grid_cap(strips * (d / 4), 256), 256, 0, ST(stream)>>>(
      g, patch_mask, (__nv_bfloat16*)dpatch_bf16, dmask_token, B, S, d, has_cls ? 1 : 0, rows_per_strip);
  return LAUNCH_RC();
}

extern "C" int mmb_split_tokens_cast(const float* g, void* a_bf16, void* b_bf16, int B, int Sa, int Sb, int d,
                                     int has_cls, void* stream) {
  if ((d & 3) || B <= 0 || Sa < 0 || Sb < 0) return MMB_ERR_ARG;
  if (Sa + Sb == 0) return MMB_OK;
  split_tokens_cast_kernel<<<grid_cap((long long)B * (Sa + Sb) * d / 4, 256), 256, 0, ST(stream)>>>(
      g, (__nv_bfloat16*)a_bf16, (__nv_bfloat16*)b_bf16, B, Sa, Sb, d, has_cls ? 1 : 0);
  return LAUNCH_RC();
}

extern "C" int mmb_tanh_bwd(const float* dy, const float* y, float* dx, void* dx_bf16, long long n, void* stream) {
  if (n <= 0) return MMB_OK;
  tanh_bwd_kernel<<<grid_cap(n, 256), 256, 0, ST(stream)>>>(dy, y, dx, (__nv_bfloat16*)dx_bf16, n);
  return LAUNCH_RC();
}

extern "C" int mmb_scatter_rows_add(const float* src, float* dst, int B, int rows_per_group, int row, int d,
                                    void* stream) {
  if ((d & 3) || B <= 0 || row < 0 || row >= rows_per_group) return MMB_ERR_ARG;
  scatter_rows_add_kernel<<<grid_cap((long long)B * d / 4, 256), 256, 0, ST(stream)>>>(src, dst, B, rows_per_group, row, d);
  return LAUNCH_RC();
}

extern "C" int mmb_scatter_rows_idx_add(const float* src, const long long* idx, float* dst, long long ld, int n, int d,
                                        void* stream) {
  if ((d & 3) || (ld & 3) || n < 0) return MMB_ERR_ARG;
  if (n == 0) return MMB_OK;
  scatter_rows_idx_add_kernel<<<grid_cap((long long)n * d / 4, 256), 256, 0, ST(stream)>>>(src, idx, dst, ld, n, d);
  return LAUNCH_RC();
}

extern "C" int mmb_ce_labels_bwd(const float* logits, long long ld, const long long* labels, long long label_stride,
                                 long long ignore_index, int M, int V, const float* accum, float grad_scale,
                                 const float* grad_scale_dev, void* dlogits_bf16, long long ldd, void* stream) {
  if (M <= 0 || V <= 0) return MMB_ERR_ARG;
  ce_labels_bwd_kernel<<<M, 256, 0, ST(stream)>>>(logits, ld, labels, label_stride, ignore_index, V, accum, grad_scale,
                                                  grad_scale_dev, (__nv_bfloat16*)dlogits_bf16, ldd);
  return LAUNCH_RC();
}

extern "C" int mmb_act_bwd(const void* dy_bf16, const void* pre_bf16, void* dx_bf16, long long n, int kind, void* stream) {
  if (n <= 0) return MMB_OK;
  if ((reinterpret_cast<uintptr_t>(dy_bf16) | reinterpret_cast<uintptr_t>(pre_bf16) | reinterpret_cast<uintptr_t>(dx_bf16)) & 3)
    return MMB_ERR_ARG;
  const __nv_bfloat16 *dy = (const __nv_bfloat16*)dy_bf16, *pre = (const __nv_bfloat16*)pre_bf16;
  if (kind == ACT_QUICK_GELU) act_bwd_kernel<0><<<grid_cap(n / 2 + 1, 256), 256, 0, ST(stream)>>>(dy, pre, (__nv_bfloat16*)dx_bf16, n);
  else if (kind == ACT_GELU_ERF) act_bwd_kernel<1><<<grid_cap(n / 2 + 1, 256), 256, 0, ST(stream)>>>(dy, pre, (__nv_bfloat16*)dx_bf16, n);
  else if (kind == ACT_RELU) act_bwd_kernel<2><<<grid_cap(n / 2 + 1, 256), 256, 0, ST(stream)>>>(dy, pre, (__nv_bfloat16*)dx_bf16, n);
  else return MMB_ERR_ARG;
  return LAUNCH_RC();
}
