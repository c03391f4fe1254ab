// HBM-bound kernels of the dual-encoder path: casts, patch im2col, token assembly, (residual-add +) LayerNorm
// forward/backward, embedding gather/scatter, L2 normalise, column sums, fused AdamW.
// All are coalesced 128-bit accesses, one warp per row for the row-wise ops, grids sized in multiples of the SM count
// for the grid-stride ones.
#include "common.cuh"
#include "mmb200_internal.h"
#include <mutex>

namespace mmb {

// ---------------------------------------------------------------------------------------------
// Deterministic reductions (mmb200_internal.h)
// ---------------------------------------------------------------------------------------------
struct ScratchEntry { int dev; cudaStream_t stream; int slot; void* ptr; size_t cap; };
static ScratchEntry g_scratch[256];
static int g_scratch_n = 0;
static std::mutex g_scratch_mu;

void* scratch(int slot, size_t bytes, cudaStream_t stream) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lk(g_scratch_mu);
  ScratchEntry* e = nullptr;
  for (int i = 0; i < g_scratch_n; ++i)
    if (g_scratch[i].dev == dev && g_scratch[i].stream == stream && g_scratch[i].slot == slot) { e = &g_scratch[i]; break; }
  if (!e) {
    if (g_scratch_n == 256) return nullptr;
    e = &g_scratch[g_scratch_n++];
    *e = ScratchEntry{dev, stream, slot, nullptr, 0};
  }
  if (bytes > e->cap) {
    if (e->ptr) cudaFree(e->ptr);
    e->ptr = nullptr; e->cap = 0;
    if (cudaMalloc(&e->ptr, bytes) != cudaSuccess) { e->ptr = nullptr; return nullptr; }
    e->cap = bytes;
  }
  return e->ptr;
}

// block = 8 row groups x 32 columns; row group r sums rows r, r+8, r+16, ... in order, then the 8 group sums are added
// in order: a fixed summation tree for every (P, N)
__global__ void __launch_bounds__(256) reduce_partials_kernel(const float* __restrict__ part, int P, int N, long long ldp,
                                                              float* __restrict__ out, int accumulate) {
  const int col = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int n = blockIdx.x * 32 + col;
  float acc = 0.f;
  if (n < N)
    for (int p = rg; p < P; p += 8) acc += part[(long long)p * ldp + n];
  __shared__ float s[8][33];
  s[rg][col] = acc;
  __syncthreads();
  if (rg == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int r = 0; r < 8; ++r) t += s[r][col];
    out[n] = accumulate ? out[n] + t : t;
  }
}

int reduce_partials(const float* part, int P, int N, long long ldp, float* out, int accumulate, cudaStream_t stream) {
  if (P <= 0 || N <= 0) return MMB_OK;
  reduce_partials_kernel<<<(N + 31) / 32, 256, 0, stream>>>(part, P, N, ldp, out, accumulate);
  return (int)cudaGetLastError();
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

static inline int grid_for(long long n_items, int per_block) {
  long long b = (n_items + per_block - 1) / per_block;
  long long cap = (long long)num_sms() * 16;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

// ---------------------------------------------------------------------------------------------
// fp32 -> bf16 cast (weights, once per optimizer step)
// SCALED: dst[i] = bf16(fl32(scale[i / per_scale] * src[i])), per_scale % 4 == 0 (the stochastic-depth factor of a
// residual-stream gradient entering the last layer's MLP branch when no final LayerNorm produces it)
// ---------------------------------------------------------------------------------------------
template <bool SCALED>
__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n,
                                     const float* __restrict__ scale, long long per_scale) {
  const long long n4 = n >> 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = __ldg(reinterpret_cast<const float4*>(src) + i);
    if (SCALED) {
      const float sc = __ldg(scale + (i << 2) / per_scale);
      v.x = __fmul_rn(sc, v.x); v.y = __fmul_rn(sc, v.y); v.z = __fmul_rn(sc, v.z); v.w = __fmul_rn(sc, v.w);
    }
    uint2 o;
    o.x = pack_bf16x2(v.x, v.y);
    o.y = pack_bf16x2(v.z, v.w);
    reinterpret_cast<uint2*>(dst)[i] = o;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long e = (n4 << 2) + threadIdx.x;
    dst[e] = __float2bfloat16(SCALED ? __fmul_rn(__ldg(scale + e / per_scale), src[e]) : src[e]);
  }
}

// bf16 -> fp32 (the bf16-compressed gradient all-reduce hands its result back to the fp32 optimizer input)
__global__ void cast_bf16_f32_kernel(const __nv_bfloat16* __restrict__ src, float* __restrict__ dst, long long n) {
  const long long n4 = n >> 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const uint2 v = __ldg(reinterpret_cast<const uint2*>(src) + i);
    reinterpret_cast<float4*>(dst)[i] = make_float4(bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y));
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) dst[(n4 << 2) + threadIdx.x] = __bfloat162float(src[(n4 << 2) + threadIdx.x]);
}

// ---------------------------------------------------------------------------------------------
// Patch im2col + cast: image [B,3,H,W] fp32 -> patches [B*P, 3*ps*ps] bf16, K order (c, kh, kw) == the flattening
// of conv.weight [width,3,ps,ps] (models/clip/image_encoder.py:50-56,91).  Patch index row-major (py, px)
// == flatten(2) of the conv output (:94).  ps must be a multiple of 2.
// ---------------------------------------------------------------------------------------------
__global__ void im2col_kernel(const float* __restrict__ img, __nv_bfloat16* __restrict__ out, int B, int H, int W,
                              int ps, long long ld_out) {
  const int gp = W / ps, P = (H / ps) * gp, K = 3 * ps * ps;
  const long long total2 = (long long)B * P * K / 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total2;
       i += (long long)gridDim.x * blockDim.x) {
    const long long e = i * 2;
    const int k = (int)(e % K);
    const long long row = e / K;
    const int p = (int)(row % P);
    const int b = (int)(row / P);
    const int c = k / (ps * ps), r = k % (ps * ps), kh = r / ps, kw = r % ps;
    const int py = p / gp, px = p % gp;
    const float2 v = __ldg(reinterpret_cast<const float2*>(
        img + (((long long)b * 3 + c) * H + (py * ps + kh)) * W + px * ps + kw));
    *reinterpret_cast<uint32_t*>(out + row * ld_out + k) = pack_bf16x2(v.x, v.y);
  }
}

// ---------------------------------------------------------------------------------------------
// Row-wise LayerNorm machinery: one warp per row, row held in registers as float4 x NV (d = 128*NV, NV <= 8).
// ---------------------------------------------------------------------------------------------
constexpr int LN_MAX_NV = 8;

struct LnRow {
  float4 v[LN_MAX_NV];
};

__device__ __forceinline__ void ln_stats(const LnRow& r, int nv, int d, float eps, float& mean, float& rstd) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_NV; ++i)
    if (i < nv) s += r.v[i].x + r.v[i].y + r.v[i].z + r.v[i].w;
  mean = warp_sum(s) / d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_NV; ++i)
    if (i < nv) {
      const float a = r.v[i].x - mean, b = r.v[i].y - mean, c = r.v[i].z - mean, e = r.v[i].w - mean;
      q += a * a + b * b + c * c + e * e;
    }
  rstd = rsqrtf(warp_sum(q) / d + eps);
}

// x_out = x_in (+ y);  ln_out = LN(x_out) * gamma + beta   (fp32 statistics, eps inside the sqrt)
//   x_in : fp32 [M,d] or nullptr;  y : bf16 [M,d] or nullptr;  x_out : fp32 [M,d] or nullptr (may alias x_in)
//   ln_bf16 : bf16 [M,d] or nullptr; ln_f32 : fp32 [M,d] or nullptr; mean/rstd : fp32 [M] or nullptr
//   row_idx : optional gather: logical row m reads physical row (m*rows_per_group + row_idx[m]) (row_idx null -> +0)
//   SCALED  : stochastic depth (torchvision stochastic_depth, mode "row"): x_out = x_in + fl32(s * y) with
//             s = scale[m / rows_per_scale] (0 or 1/(1-p) per sample, drawn on the host side); no gather mode.
// Replaces F.layer_norm + residual add (torch/nn/modules/transformer.py:946-951) and Fp32LayerNorm
// (torchmultimodal/modules/layers/normalizations.py:17-25).
template <bool SCALED>
__global__ void add_ln_fwd_kernel(const float* __restrict__ x_in, const __nv_bfloat16* __restrict__ y,
                                  float* __restrict__ x_out, __nv_bfloat16* __restrict__ ln_bf16,
                                  float* __restrict__ ln_f32, const float* __restrict__ gamma,
                                  const float* __restrict__ beta, float* __restrict__ mean_out,
                                  float* __restrict__ rstd_out, const int* __restrict__ row_idx, int rows_per_group,
                                  int M, int d, float eps, const float* __restrict__ scale, int rows_per_scale) {
  const int nv = d >> 7;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int m = blockIdx.x * wpb + (threadIdx.x >> 5); m < M; m += gridDim.x * wpb) {
    long long src = m;
    if (rows_per_group > 0) src = (long long)m * rows_per_group + (row_idx ? row_idx[m] : 0);
    float s = 1.f;
    if (SCALED) s = __ldg(scale + m / rows_per_scale);
    LnRow r;
#pragma unroll
    for (int i = 0; i < LN_MAX_NV; ++i)
      if (i < nv) {
        const int c = (i * 32 + lane) * 4;
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        if (x_in) a = *reinterpret_cast<const float4*>(x_in + src * d + c);
        if (y) {
          const uint2 u = *reinterpret_cast<const uint2*>(y + src * d + c);
          if (SCALED) {  // the product is rounded on its own (no FMA), as input * noise is in the reference
            a.x += __fmul_rn(s, bf16_lo(u.x)); a.y += __fmul_rn(s, bf16_hi(u.x));
            a.z += __fmul_rn(s, bf16_lo(u.y)); a.w += __fmul_rn(s, bf16_hi(u.y));
          } else {
            a.x += bf16_lo(u.x); a.y += bf16_hi(u.x); a.z += bf16_lo(u.y); a.w += bf16_hi(u.y);
          }
        }
        r.v[i] = a;
        if (x_out) *reinterpret_cast<float4*>(x_out + (long long)m * d + c) = a;  // compact in gather mode
      }
    float mean, rstd;
    ln_stats(r, nv, d, eps, mean, rstd);
    if (lane == 0) {
      if (mean_out) mean_out[m] = mean;
      if (rstd_out) rstd_out[m] = rstd;
    }
#pragma unroll
    for (int i = 0; i < LN_MAX_NV; ++i)
      if (i < nv) {
        const int c = (i * 32 + lane) * 4;
        const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
        const float4 b = __ldg(reinterpret_cast<const float4*>(beta + c));
        float4 o;
        o.x = (r.v[i].x - mean) * rstd * g.x + b.x;
        o.y = (r.v[i].y - mean) * rstd * g.y + b.y;
        o.z = (r.v[i].z - mean) * rstd * g.z + b.z;
        o.w = (r.v[i].w - mean) * rstd * g.w + b.w;
        if (ln_bf16) {
          uint2 u;
          u.x = pack_bf16x2(o.x, o.y);
          u.y = pack_bf16x2(o.z, o.w);
          *reinterpret_cast<uint2*>(ln_bf16 + (long long)m * d + c) = u;
        }
        if (ln_f32) *reinterpret_cast<float4*>(ln_f32 + (long long)m * d + c) = o;
      }
  }
}

// CLIP ViT token assembly + ln_pre (models/clip/image_encoder.py:94-106):
//   t[b,0,:] = cls + pos[0];  t[b,1+p,:] = patch_out[b*P+p,:] + pos[1+p];  x0 = Fp32LayerNorm(t)
// patch_out is the bf16 output of the patch-embedding GEMM.  Saves mean/rstd of t for the backward.
__global__ void vit_embed_ln_fwd_kernel(const __nv_bfloat16* __restrict__ patch_out, const float* __restrict__ cls,
                                        const float* __restrict__ pos, const float* __restrict__ gamma,
                                        const float* __restrict__ beta, float* __restrict__ x0,
                                        float* __restrict__ mean_out, float* __restrict__ rstd_out, int B, int S,
                                        int d, float eps) {
  const int nv = d >> 7;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int M = B * S;
  for (int m = blockIdx.x * wpb + (threadIdx.x >> 5); m < M; m += gridDim.x * wpb) {
    const int b = m / S, s = m - b * S;
    LnRow r;
#pragma unroll
    for (int i = 0; i < LN_MAX_NV; ++i)
      if (i < nv) {
        const int c = (i * 32 + lane) * 4;
        float4 a = __ldg(reinterpret_cast<const float4*>(pos + (long long)s * d + c));
        if (s == 0) {
          const float4 t = __ldg(reinterpret_cast<const float4*>(cls + c));
          a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
        } else {
          const uint2 u = *reinterpret_cast<const uint2*>(patch_out + ((long long)b * (S - 1) + (s - 1)) * d + c);
          a.x += bf16_lo(u.x); a.y += bf16_hi(u.x); a.z += bf16_lo(u.y); a.w += bf16_hi(u.y);
        }
        r.v[i] = a;
      }
    float mean, rstd;
    ln_stats(r, nv, d, eps, mean, rstd);
    if (lane == 0) { mean_out[m] = mean; rstd_out[m] = rstd; }
#pragma unroll
    for (int i = 0; i < LN_MAX_NV; ++i)
      if (i < nv) {
        const int c = (i * 32 + lane) * 4;
        const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
        const float4 bb = __ldg(reinterpret_cast<const float4*>(beta + c));
        float4 o;
        o.x = (r.v[i].x - mean) * rstd * g.x + bb.x;
        o.y = (r.v[i].y - mean) * rstd * g.y + bb.y;
        o.z = (r.v[i].z - mean) * rstd * g.z + bb.z;
        o.w = (r.v[i].w - mean) * rstd * g.w + bb.w;
        *reinterpret_cast<float4*>(x0 + (long long)m * d + c) = o;
      }
  }
}

// BERT embeddings (modules/layers/text_embedding.py:70-104): x = LayerNorm(word[ids] + pos[s] + type[type_ids]),
// position ids = arange(S), token types default to 0.  One warp per token, fp32 statistics.
__global__ void bert_embed_ln_fwd_kernel(const long long* __restrict__ ids, const long long* __restrict__ type_ids,
                                         const float* __restrict__ word, const float* __restrict__ pos,
                                         const float* __restrict__ type, const float* __restrict__ gamma,
                                         const float* __restrict__ beta, float* __restrict__ x,
                                         unsigned char* __restrict__ kmask_out, long long pad_id, int B, int S, int d,
                                         int V, float eps) {
  const int nv = d >> 7;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int M = B * S;
  for (int m = blockIdx.x * wpb + (threadIdx.x >> 5); m < M; m += gridDim.x * wpb) {
    const int s = m % S;
    const long long tok = ids[m];
    if (tok < 0 || tok >= V) __trap();
    const long long ty = type_ids ? type_ids[m] : 0;
    if (kmask_out && lane == 0) kmask_out[m] = (tok != pad_id) ? 1 : 0;  // bert_text_encoder.py:87-90 (bit-exact)
    LnRow r;
#pragma unroll
    for (int i = 0; i < LN_MAX_NV; ++i)
      if (i < nv) {
        const int c = (i * 32 + lane) * 4;
        const float4 a = __ldg(reinterpret_cast<const float4*>(word + tok * d + c));
        const float4 b = __ldg(reinterpret_cast<const float4*>(pos + (long long)s * d + c));
        const float4 t = __ldg(reinterpret_cast<const float4*>(type + ty * d + c));
        r.v[i] = make_float4(a.x + b.x + t.x, a.y + b.y + t.y, a.z + b.z + t.z, a.w + b.w + t.w);
      }
    float mean, rstd;
    ln_stats(r, nv, d, eps, mean, rstd);
#pragma unroll
    for (int i = 0; i < LN_MAX_NV; ++i)
      if (i < nv) {
        const int c = (i * 32 + lane) * 4;
        const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
        const float4 bb = __ldg(reinterpret_cast<const float4*>(beta + c));
        float4 o;
        o.x = (r.v[i].x - mean) * rstd * g.x + bb.x;
        o.y = (r.v[i].y - mean) * rstd * g.y + bb.y;
        o.z = (r.v[i].z - mean) * rstd * g.z + bb.z;
        o.w = (r.v[i].w - mean) * rstd * g.w + bb.w;
        *reinterpret_cast<float4*>(x + (long long)m * d + c) = o;
      }
  }
}

// ViT token assembly without LayerNorm (FLAVA: models/flava/image_encoder.py:139-175; TorchMultimodal PatchEmbeddings:
// modules/layers/patch_embedding.py:104-154):  with cls:  x[b,0] = cls + pos[0]; x[b,1+p] = e[b,p] + pos[1+p]
//                                             cls == NULL (CoCa, include_cls_embed=False): x[b,p] = e[b,p] + pos[p]
// where e[b,p] = mask[b,p] ? mask_token : patch_out[b*P+p].
__global__ void vit_assemble_fwd_kernel(const __nv_bfloat16* __restrict__ patch_out, const float* __restrict__ cls,
                                        const float* __restrict__ pos, const float* __restrict__ mask_token,
                                        const unsigned char* __restrict__ patch_mask, float* __restrict__ x, int B, int S,
                                        int d) {
  const int d4 = d >> 2;
  const int off = cls ? 1 : 0, P = S - off;
  const long long total = (long long)B * S * d4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d4) * 4;
    const long long row = i / d4;
    const int s = (int)(row % S);
    const int b = (int)(row / S);
    float4 a = __ldg(reinterpret_cast<const float4*>(pos + (long long)s * d + c));
    float4 t;
    if (s < off) {
      t = __ldg(reinterpret_cast<const float4*>(cls + c));
    } else if (patch_mask && mask_token && patch_mask[(long long)b * P + (s - off)]) {
      t = __ldg(reinterpret_cast<const float4*>(mask_token + c));
    } else {
      const uint2 u = *reinterpret_cast<const uint2*>(patch_out + ((long long)b * P + (s - off)) * d + c);
      t = make_float4(bf16_lo(u.x), bf16_hi(u.x), bf16_lo(u.y), bf16_hi(u.y));
    }
    reinterpret_cast<float4*>(x)[i] = make_float4(a.x + t.x, a.y + t.y, a.z + t.z, a.w + t.w);
  }
}

// CoCa text embeddings (models/coca/text_decoder.py:48-60): x[b,s] = emb[ids[b,s]] + pos[s] for s < S-1 and
// x[b,S-1] = cls + pos[S-1] (the CLS embedding is appended, not prepended).  cls == NULL: plain S-token embedding.
__global__ void coca_text_embed_fwd_kernel(const long long* __restrict__ ids, const float* __restrict__ emb,
                                           const float* __restrict__ cls, const float* __restrict__ pos,
                                           float* __restrict__ x, int B, int S, int d, int V) {
  const int d4 = d >> 2;
  const int T = cls ? S - 1 : S;  // tokens per sequence in ids
  const long long total = (long long)B * S * d4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d4);
    const long long row = i / d4;
    const int s = (int)(row % S);
    const long long b = row / S;
    float4 e;
    if (s < T) {
      const long long tok = ids[b * T + s];
      if (tok < 0 || tok >= V) __trap();
      e = __ldg(reinterpret_cast<const float4*>(emb + tok * d) + c);
    } else {
      e = __ldg(reinterpret_cast<const float4*>(cls) + c);
    }
    const float4 p = __ldg(reinterpret_cast<const float4*>(pos + (long long)s * d) + c);
    reinterpret_cast<float4*>(x)[i] = make_float4(e.x + p.x, e.y + p.y, e.z + p.z, e.w + p.w);
  }
}

// Cross-entropy over rows of fp32 logits [M, V] against int64 labels with ignore_index (nn.CrossEntropyLoss(
// ignore_index=pad) of models/coca/coca_model.py:425,447-450): accum[0] += sum of row losses, accum[1] += #valid rows
// (row i writes (loss, 1) or (0, 0) to part2[2i..]; the host wrapper sums them in row order).
__global__ void __launch_bounds__(256) ce_labels_kernel(const float* __restrict__ logits, long long ld,
                                                        const long long* __restrict__ labels, long long label_stride,
                                                        long long ignore_index, int M, int V,
                                                        float* __restrict__ row_loss, float* __restrict__ part2) {
  __shared__ float red[8];
  const int i = blockIdx.x;
  if (i >= M) return;
  const long long lab = labels[(long long)i * label_stride];
  if (lab == ignore_index) {
    if (threadIdx.x == 0) {
      if (row_loss) row_loss[i] = 0.f;
      part2[2 * i] = 0.f; part2[2 * i + 1] = 0.f;
    }
    return;
  }
  if (lab < 0 || lab >= V) __trap();
  const float* row = logits + (long long)i * ld;
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < V; j += blockDim.x) mx = fmaxf(mx, row[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float se = 0.f;
  for (int j = threadIdx.x; j < V; j += blockDim.x) se += __expf(row[j] - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = se;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    const float loss = mx + logf(t) - row[lab];
    if (row_loss) row_loss[i] = loss;
    part2[2 * i] = loss; part2[2 * i + 1] = 1.f;
  }
}

// out[m,:] = bf16(x[idx[m]*ld : +d])   (boolean-mask row selects `hidden[masked_tokens, :]` of the FLAVA masked-prediction
// losses, modules/losses/flava.py:212-215, as a GEMM operand; idx = flat row numbers of the kept tokens)
__global__ void gather_rows_idx_cast_kernel(const float* __restrict__ x, long long ld, const long long* __restrict__ idx,
                                            __nv_bfloat16* __restrict__ out, int n, int d) {
  const int d4 = d >> 2;
  const long long total = (long long)n * d4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d4) * 4;
    const long long m = i / d4;
    const float4 v = *reinterpret_cast<const float4*>(x + idx[m] * ld + c);
    uint2 u;
    u.x = pack_bf16x2(v.x, v.y);
    u.y = pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(out + m * d + c) = u;
  }
}

// out[b,:] = bf16(x[(b*rows_per_group + row)*d : +d])   (select one token per sequence, e.g. CLS, as a GEMM operand)
__global__ void gather_rows_cast_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out, int B,
                                        int rows_per_group, int row, int d) {
  const int d4 = d >> 2;
  const long long total = (long long)B * d4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d4) * 4;
    const long long b = i / d4;
    const float4 v = *reinterpret_cast<const float4*>(x + (b * rows_per_group + row) * d + c);
    uint2 u;
    u.x = pack_bf16x2(v.x, v.y);
    u.y = pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(out + b * d + c) = u;
  }
}

__global__ void tanh_inplace_kernel(float* __restrict__ x, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    x[i] = tanhf(x[i]);
}

// out[b] = cat(cls (optional), a[b], b[b]) along the sequence dim; all fp32 [.., d]
// (FLAVATransformerWithoutEmbeddings.forward + FLAVAModel.encode_mm: models/flava/transformer.py:55-58, model.py:294-297)
__global__ void concat_tokens_kernel(const float* __restrict__ cls, const float* __restrict__ a,
                                     const float* __restrict__ bsrc, float* __restrict__ out, int B, int Sa, int Sb,
                                     int d) {
  const int d4 = d >> 2;
  const int So = (cls ? 1 : 0) + Sa + Sb;
  const long long total = (long long)B * So * d4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d4) * 4;
    const long long row = i / d4;
    int s = (int)(row % So);
    const long long b = row / So;
    float4 v;
    if (cls) {
      if (s == 0) { reinterpret_cast<float4*>(out)[i] = __ldg(reinterpret_cast<const float4*>(cls + c)); continue; }
      s -= 1;
    }
    if (s < Sa) v = *reinterpret_cast<const float4*>(a + (b * Sa + s) * d + c);
    else        v = *reinterpret_cast<const float4*>(bsrc + (b * Sb + (s - Sa)) * d + c);
    reinterpret_cast<float4*>(out)[i] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// LayerNorm backward (+ residual-gradient add).  For each row:
//   xhat = (x - mean) * rstd;  dyg = dy * gamma
//   dx   = rstd * (dyg - mean_d(dyg) - xhat * mean_d(dyg * xhat))
//   g_out = (g_in ? g_in : 0) + dx         (fp32 [M,d], may alias g_in)     and/or  g_bf16 = bf16(g_out)
//   SCALED (stochastic depth of the branch that reads g_bf16): g_bf16 = bf16(fl32(s * g_out)),
//   s = scale[m / rows_per_scale]; gsum sums those scaled bf16 values; g_out is unscaled (the residual path)
//   dgamma += sum_rows dy * xhat ; dbeta += sum_rows dy      (fp32 atomics, one per column per block)
// Input modes for x:  MODE_X      : x fp32 [M,d]
//                     MODE_VIT    : x is re-assembled from patch_out/cls/pos (token assembly, see above)
// dy is bf16 [M,d] (dy_bf16) or fp32 [M,d] (dy_f32).  Row scatter: with row_idx/rows_per_group the logical row m
// reads x and writes g at physical row m*rows_per_group + row_idx[m].
// ---------------------------------------------------------------------------------------------
struct LnBwdArgs {
  const float* x; const __nv_bfloat16* patch_out; const float* cls; const float* pos; int S;  // x sources
  const __nv_bfloat16* dy_bf16; const float* dy_f32;
  const float* mean; const float* rstd; const float* gamma;
  const float* g_in; float* g_out; __nv_bfloat16* g_bf16;
  float* dgamma; float* dbeta;
  float* gsum;  // optional: gsum[c] += sum_rows bf16(g_out[row, c]) — the bias gradient of the Linear that consumes g_bf16
  float* part;  // [3][gridDim.x][d] per-CTA column partials of dgamma / dbeta / gsum (reduced in a fixed order)
  const int* row_idx; int rows_per_group;
  int M, d;
  const float* scale; int rows_per_scale;  // SCALED only: per-sample factor of g_bf16
};

// One CTA of NV warps per row (one float4 of the row per thread): ~20 live registers per thread, so 10-16 CTAs are
// resident per SM and 60+ warps hide the HBM latency (a warp-per-row layout would keep the whole row plus three
// per-lane column accumulators in ~170 registers and leave only 12 warps per SM to hide it).
// The two row reductions cross the NV warps through a double-buffered smem slot: one __syncthreads per row.
template <bool VIT, int NV, bool SCALED>
__global__ void __launch_bounds__(NV * 32, (1536 / (NV * 32) > 32 ? 32 : 1536 / (NV * 32))) ln_bwd_kernel(const LnBwdArgs a) {
  constexpr int d = NV * 128;
  __shared__ float part[2][NV][2];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int c = threadIdx.x * 4;
  const float4 gm = __ldg(reinterpret_cast<const float4*>(a.gamma + c));
  float4 accg = make_float4(0.f, 0.f, 0.f, 0.f), accb = accg, accs = accg;
  const bool want_gsum = a.gsum != nullptr;
  int buf = 0;
  for (int m = blockIdx.x; m < a.M; m += gridDim.x) {
    long long phys = m;
    if (a.rows_per_group > 0) phys = (long long)m * a.rows_per_group + (a.row_idx ? a.row_idx[m] : 0);
    // issue every global load of the row before the first use
    float4 x, dy, gi = make_float4(0.f, 0.f, 0.f, 0.f);
    uint2 pu = make_uint2(0u, 0u), du = pu;
    float4 cl = make_float4(0.f, 0.f, 0.f, 0.f);
    int s = 0;
    if (VIT) {
      const int b = m / a.S;
      s = m - b * a.S;
      x = __ldg(reinterpret_cast<const float4*>(a.pos + (long long)s * d + c));
      if (s == 0) cl = __ldg(reinterpret_cast<const float4*>(a.cls + c));
      else pu = *reinterpret_cast<const uint2*>(a.patch_out + ((long long)b * (a.S - 1) + (s - 1)) * d + c);
    } else {
      x = *reinterpret_cast<const float4*>(a.x + (long long)m * d + c);  // compact in gather mode
    }
    if (a.dy_bf16) du = *reinterpret_cast<const uint2*>(a.dy_bf16 + (long long)m * d + c);
    else           dy = *reinterpret_cast<const float4*>(a.dy_f32 + (long long)m * d + c);
    if (a.g_in) gi = *reinterpret_cast<const float4*>(a.g_in + phys * d + c);
    const float mean = a.mean[m], rstd = a.rstd[m];
    float sc = 1.f;
    if (SCALED) sc = __ldg(a.scale + m / a.rows_per_scale);
    if (VIT) {
      if (s == 0) { x.x += cl.x; x.y += cl.y; x.z += cl.z; x.w += cl.w; }
      else { x.x += bf16_lo(pu.x); x.y += bf16_hi(pu.x); x.z += bf16_lo(pu.y); x.w += bf16_hi(pu.y); }
    }
    if (a.dy_bf16) dy = make_float4(bf16_lo(du.x), bf16_hi(du.x), bf16_lo(du.y), bf16_hi(du.y));
    float4 h;
    h.x = (x.x - mean) * rstd; h.y = (x.y - mean) * rstd; h.z = (x.z - mean) * rstd; h.w = (x.w - mean) * rstd;
    accg.x += dy.x * h.x; accg.y += dy.y * h.y; accg.z += dy.z * h.z; accg.w += dy.w * h.w;
    accb.x += dy.x; accb.y += dy.y; accb.z += dy.z; accb.w += dy.w;
    dy.x *= gm.x; dy.y *= gm.y; dy.z *= gm.z; dy.w *= gm.w;  // dy * gamma
    float s1 = warp_sum(dy.x + dy.y + dy.z + dy.w);
    float s2 = warp_sum(dy.x * h.x + dy.y * h.y + dy.z * h.z + dy.w * h.w);
    if (NV > 1) {
      if (lane == 0) { part[buf][w][0] = s1; part[buf][w][1] = s2; }
      __syncthreads();
      s1 = 0.f; s2 = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) { s1 += part[buf][i][0]; s2 += part[buf][i][1]; }
      buf ^= 1;
    }
    s1 *= (1.f / d);
    s2 *= (1.f / d);
    float4 o;
    o.x = rstd * (dy.x - s1 - h.x * s2) + gi.x;
    o.y = rstd * (dy.y - s1 - h.y * s2) + gi.y;
    o.z = rstd * (dy.z - s1 - h.z * s2) + gi.z;
    o.w = rstd * (dy.w - s1 - h.w * s2) + gi.w;
    if (a.g_out) *reinterpret_cast<float4*>(a.g_out + phys * d + c) = o;
    if (a.g_bf16) {
      uint2 u;
      if (SCALED) {
        u.x = pack_bf16x2(__fmul_rn(sc, o.x), __fmul_rn(sc, o.y));
        u.y = pack_bf16x2(__fmul_rn(sc, o.z), __fmul_rn(sc, o.w));
      } else {
        u.x = pack_bf16x2(o.x, o.y);
        u.y = pack_bf16x2(o.z, o.w);
      }
      if (want_gsum) {  // sums the ROUNDED values: identical to a column sum over the stored bf16 tensor
        accs.x += bf16_lo(u.x); accs.y += bf16_hi(u.x); accs.z += bf16_lo(u.y); accs.w += bf16_hi(u.y);
      }
      if (VIT) {  // bf16 gradient of the patch-embedding GEMM output: compact [B*(S-1), d], CLS row dropped
        const int b = m / a.S;
        if (s > 0) *reinterpret_cast<uint2*>(a.g_bf16 + ((long long)b * (a.S - 1) + (s - 1)) * d + c) = u;
      } else {
        *reinterpret_cast<uint2*>(a.g_bf16 + phys * d + c) = u;
      }
    }
  }
  // every thread owns 4 distinct columns: this CTA's partial sums, reduced across CTAs in a fixed order afterwards
  const long long plane = (long long)gridDim.x * d;
  float* pp = a.part + (long long)blockIdx.x * d + c;
  if (a.dgamma) *reinterpret_cast<float4*>(pp) = accg;
  if (a.dbeta) *reinterpret_cast<float4*>(pp + plane) = accb;
  if (want_gsum) *reinterpret_cast<float4*>(pp + 2 * plane) = accs;
}

template <bool VIT, bool SCALED = false>
static int launch_ln_bwd(LnBwdArgs a, cudaStream_t st) {
  const int nv = a.d >> 7;
  const int threads = nv * 32;
  int per_sm = 1536 / threads;   // matches the kernel's __launch_bounds__ (<= 42 registers per thread)
  if (per_sm > 24) per_sm = 24;
  int grid = num_sms() * per_sm;
  if (grid > a.M) grid = a.M;
  if (grid < 1) return MMB_ERR_ARG;
  const bool any_col = a.dgamma || a.dbeta || a.gsum;
  if (any_col) {
    a.part = static_cast<float*>(scratch(SCR_LN_BWD, 3ull * grid * a.d * sizeof(float), st));
    if (!a.part) return (int)cudaErrorMemoryAllocation;
  }
  switch (nv) {
#define LNB(NVV) case NVV: ln_bwd_kernel<VIT, NVV, SCALED><<<grid, threads, 0, st>>>(a); break;
    LNB(1) LNB(2) LNB(3) LNB(4) LNB(5) LNB(6) LNB(7) LNB(8)
#undef LNB
    default: return MMB_ERR_UNSUPPORTED;
  }
  int rc = (int)cudaGetLastError();
  const long long plane = (long long)grid * a.d;
  float* outs[3] = {a.dgamma, a.dbeta, a.gsum};
  for (int i = 0; i < 3 && rc == 0; ++i)
    if (outs[i]) rc = reduce_partials(a.part + i * plane, grid, a.d, a.d, outs[i], 1, st);
  return rc;
}

// ---------------------------------------------------------------------------------------------
// out[j] += sum_b in[b, j]   (positional-embedding / cls-token gradients: sum over the batch)
//   in fp32 [Bn, n] with row stride ld; columns [0,n) ; optional row subset via (row0, row_step)
// ---------------------------------------------------------------------------------------------
// Each blockIdx.y writes its chunk's sums to part[blockIdx.y][n]; reduce_partials adds the chunks in order.
__global__ void batch_sum_kernel(const float* __restrict__ in, float* __restrict__ part, int Bn, long long ld, int n,
                                 int b_chunk) {
  const int j = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (j >= n) return;
  const int b0 = blockIdx.y * b_chunk, b1 = min(b0 + b_chunk, Bn);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int b = b0; b < b1; ++b) {
    const float4 v = *reinterpret_cast<const float4*>(in + (long long)b * ld + j);
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  *reinterpret_cast<float4*>(part + (long long)blockIdx.y * n + j) = acc;
}

// ---------------------------------------------------------------------------------------------
// out[n] += sum_m x[m, n]   (bias gradients), x bf16 [M, N] row-major with leading dim ld
// ---------------------------------------------------------------------------------------------
// Each blockIdx.y writes its row chunk's sums to part[blockIdx.y][N]; reduce_partials adds the chunks in order.
__global__ void __launch_bounds__(256) colsum_bf16_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ part,
                                                          int M, int N, long long ld, int rows_per_block) {
  // block = 256 threads: 32 column-octets (256 columns) x 8 row lanes; 4 independent 16 B loads in flight per thread
  const int co = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int n = (blockIdx.x * 32 + co) * 8;
  const int m0 = blockIdx.y * rows_per_block, m1 = min(m0 + rows_per_block, M);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (n < N) {
    int m = m0 + rl;
    for (; m + 24 < m1; m += 32) {
      uint4 u[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(x + (long long)(m + 8 * k) * ld + n));
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        acc[0] += bf16_lo(u[k].x); acc[1] += bf16_hi(u[k].x); acc[2] += bf16_lo(u[k].y); acc[3] += bf16_hi(u[k].y);
        acc[4] += bf16_lo(u[k].z); acc[5] += bf16_hi(u[k].z); acc[6] += bf16_lo(u[k].w); acc[7] += bf16_hi(u[k].w);
      }
    }
    for (; m < m1; m += 8) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(x + (long long)m * ld + n));
      acc[0] += bf16_lo(u.x); acc[1] += bf16_hi(u.x); acc[2] += bf16_lo(u.y); acc[3] += bf16_hi(u.y);
      acc[4] += bf16_lo(u.z); acc[5] += bf16_hi(u.z); acc[6] += bf16_lo(u.w); acc[7] += bf16_hi(u.w);
    }
  }
  __shared__ float s[8][32][9];
#pragma unroll
  for (int e = 0; e < 8; ++e) s[rl][co][e] = acc[e];
  __syncthreads();
  if (rl == 0 && n < N) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float t = 0.f;
#pragma unroll
      for (int r = 0; r < 8; ++r) t += s[r][co][e];
      part[(long long)blockIdx.y * N + n + e] = t;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Text embedding: x[b,s,:] = emb[token[b,s],:] + pos[s,:]   (models/clip/text_encoder.py:118-119)
// Token ids are int64 (bit-exact gather); ids outside [0,V) trap (torch raises an index error).
// ---------------------------------------------------------------------------------------------
__global__ void text_embed_fwd_kernel(const long long* __restrict__ tokens, const float* __restrict__ emb,
                                      const float* __restrict__ pos, float* __restrict__ x, int B, int S, int d,
                                      int V) {
  const int d4 = d >> 2;
  const long long total = (long long)B * S * d4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d4);
    const long long row = i / d4;
    const int s = (int)(row % S);
    const long long tok = tokens[row];
    if (tok < 0 || tok >= V) __trap();
    const float4 e = __ldg(reinterpret_cast<const float4*>(emb + tok * d) + c);
    const float4 p = __ldg(reinterpret_cast<const float4*>(pos + (long long)s * d) + c);
    reinterpret_cast<float4*>(x)[i] = make_float4(e.x + p.x, e.y + p.y, e.z + p.z, e.w + p.w);
  }
}
// demb[token[b,s],:] += g[b,s,:]  (dpos is produced by batch_sum).  Deterministic without atomics: CTA k owns the
// token ids t with t % gridDim.x == k, walks all B*S rows in order (a ballot per 32 rows finds its own) and adds
// each of its rows into the table with plain read-modify-writes, so every table row is summed in row order by one CTA.
__global__ void __launch_bounds__(256) text_embed_bwd_kernel(const long long* __restrict__ tokens, const float* __restrict__ g,
                                                             float* __restrict__ demb, int rows, int d) {
  __shared__ long long tok[256];
  __shared__ unsigned mask[8];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int d4 = d >> 2;
  for (int r0 = 0; r0 < rows; r0 += 256) {
    const int r = r0 + threadIdx.x;
    const long long t = r < rows ? tokens[r] : -1;
    const bool mine = r < rows && (int)((unsigned long long)t % gridDim.x) == (int)blockIdx.x;
    tok[threadIdx.x] = t;
    const unsigned m = __ballot_sync(0xffffffffu, mine);
    if (lane == 0) mask[w] = m;
    __syncthreads();
    for (int ww = 0; ww < 8; ++ww) {
      unsigned mm = mask[ww];
      while (mm) {
        const int i = ww * 32 + __ffs(mm) - 1;
        mm &= mm - 1;
        const float4* src = reinterpret_cast<const float4*>(g + (long long)(r0 + i) * d);
        float4* dst = reinterpret_cast<float4*>(demb + tok[i] * d);
        for (int c = threadIdx.x; c < d4; c += blockDim.x) {
          const float4 v = src[c];
          float4 o = dst[c];
          o.x += v.x; o.y += v.y; o.z += v.z; o.w += v.w;
          dst[c] = o;
        }
      }
    }
    __syncthreads();
  }
}
// idx[b] = argmax_s tokens[b,s] (first maximum, like torch.argmax)  (models/clip/text_encoder.py:130-132)
__global__ void argmax_tokens_kernel(const long long* __restrict__ tokens, int* __restrict__ idx, int B, int S) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= B) return;
  long long best = LLONG_MIN;
  int bi = 0x7fffffff;
  for (int s = lane; s < S; s += 32) {
    const long long t = tokens[(long long)b * S + s];
    if (t > best) { best = t; bi = s; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const long long ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  if (lane == 0) idx[b] = bi;
}

// ---------------------------------------------------------------------------------------------
// L2 normalise rows (F.normalize, models/clip/model.py:72-73): y = x / max(||x||, eps)
// ---------------------------------------------------------------------------------------------
__global__ void l2norm_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, __nv_bfloat16* __restrict__ y_bf16,
                                  float* __restrict__ inv_norm, int B, int E, float eps) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= B) return;
  float s = 0.f;
  for (int c = lane; c < E; c += 32) {
    const float v = x[(long long)b * E + c];
    s += v * v;
  }
  s = warp_sum(s);
  const float inv = 1.f / fmaxf(sqrtf(s), eps);
  if (lane == 0 && inv_norm) inv_norm[b] = inv;
  for (int c = lane; c < E; c += 32) {
    const float o = x[(long long)b * E + c] * inv;
    if (y) y[(long long)b * E + c] = o;
    if (y_bf16) y_bf16[(long long)b * E + c] = __float2bfloat16(o);
  }
}
// dx = (dy - y * <y, dy>) * inv_norm     (valid when ||x|| > eps, which holds for any non-degenerate embedding)
__global__ void l2norm_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y,
                                  const float* __restrict__ inv_norm, float* __restrict__ dx,
                                  __nv_bfloat16* __restrict__ dx_bf16, int B, int E) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= B) return;
  float s = 0.f;
  for (int c = lane; c < E; c += 32) s += dy[(long long)b * E + c] * y[(long long)b * E + c];
  s = warp_sum(s);
  const float inv = inv_norm[b];
  for (int c = lane; c < E; c += 32) {
    const float o = (dy[(long long)b * E + c] - y[(long long)b * E + c] * s) * inv;
    if (dx) dx[(long long)b * E + c] = o;
    if (dx_bf16) dx_bf16[(long long)b * E + c] = __float2bfloat16(o);
  }
}

// ---------------------------------------------------------------------------------------------
// Fused AdamW over a flat parameter buffer (torch.optim.AdamW semantics, decoupled weight decay); also emits the
// bf16 copy of the updated weights that the next step's GEMMs read, and zeroes the gradient.
// ---------------------------------------------------------------------------------------------
__global__ void adamw_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                             __nv_bfloat16* __restrict__ p_bf16, long long n, float lr, float beta1, float beta2,
                             float eps, float wd, float bc1, float bc2, float grad_scale, int zero_grad) {
  const long long n4 = n >> 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 P = reinterpret_cast<float4*>(p)[i];
    float4 G = reinterpret_cast<float4*>(g)[i];
    float4 Mv = reinterpret_cast<float4*>(m)[i];
    float4 V = reinterpret_cast<float4*>(v)[i];
    float* pp = &P.x; float* gg = &G.x; float* mm = &Mv.x; float* vv = &V.x;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float gr = gg[e] * grad_scale;
      pp[e] *= (1.f - lr * wd);
      mm[e] = beta1 * mm[e] + (1.f - beta1) * gr;
      vv[e] = beta2 * vv[e] + (1.f - beta2) * gr * gr;
      const float denom = sqrtf(vv[e]) / sqrtf(bc2) + eps;
      pp[e] -= (lr / bc1) * (mm[e] / denom);
    }
    reinterpret_cast<float4*>(p)[i] = P;
    reinterpret_cast<float4*>(m)[i] = Mv;
    reinterpret_cast<float4*>(v)[i] = V;
    if (zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p_bf16) {
      uint2 u;
      u.x = pack_bf16x2(P.x, P.y);
      u.y = pack_bf16x2(P.z, P.w);
      reinterpret_cast<uint2*>(p_bf16)[i] = u;
    }
  }
}


// ---------------------------------------------------------------------------------------------
// AnyPrecisionAdamW (torchmultimodal/modules/optimizers/anyprecision.py:99-199): AdamW whose momentum, variance and
// Kahan-compensation buffers live in caller-chosen dtypes (fp32 or bf16; reference defaults: fp32 momentum, bf16
// variance, bf16 compensation).  Every in-place op of the reference rounds to the STATE's dtype; the kernel reproduces
// those roundings one for one (rn<T>) with fp32 op-math in between, as TensorIterator does for mixed-dtype operands:
//   m  = rn_M(rn_M(m * b1) + (1 - b1) * g)                      (:161  mul_ ; add_(alpha))
//   v  = rn_V(fma((1 - b2) * g, g, rn_V(v * b2)))               (:164  mul_ ; addcmul_)
//   cv = rn_V(rn_V(rn_V(sqrt(v)) / sqrt(1 - b2^t)) + eps)       (:174  sqrt ; / ; add_)
//   plain: p += -step_size * (m / cv)                           (:190  addcdiv_)
//   Kahan: c = rn_C(c - step_size * (m / cv)); t = p; p += c; c = rn_C(c + (t - p))      (:177-186)
// Parameters and gradients are fp32 (this runtime keeps fp32 masters); the bf16 GEMM shadow is refreshed in the same
// pass.  One fused pass instead of the reference's ~12 elementwise kernels per parameter tensor.
// ---------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ float st_load(const T* p, long long i);
template <> __device__ __forceinline__ float st_load<float>(const float* p, long long i) { return p[i]; }
template <> __device__ __forceinline__ float st_load<__nv_bfloat16>(const __nv_bfloat16* p, long long i) { return __bfloat162float(p[i]); }
template <typename T> __device__ __forceinline__ float rn(float x);
template <> __device__ __forceinline__ float rn<float>(float x) { return x; }
template <> __device__ __forceinline__ float rn<__nv_bfloat16>(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
template <typename T> __device__ __forceinline__ void st_store(T* p, long long i, float x);
template <> __device__ __forceinline__ void st_store<float>(float* p, long long i, float x) { p[i] = x; }
template <> __device__ __forceinline__ void st_store<__nv_bfloat16>(__nv_bfloat16* p, long long i, float x) { p[i] = __float2bfloat16_rn(x); }

template <typename TM, typename TV, typename TC, bool KAHAN>
__global__ void anyprecision_adamw_kernel(float* __restrict__ p, float* __restrict__ g, TM* __restrict__ m,
                                          TV* __restrict__ v, TC* __restrict__ comp, __nv_bfloat16* __restrict__ p_bf16,
                                          long long n, float decay, float beta1, float beta2, float alpha1, float alpha2,
                                          float eps, float neg_step_size, float denom_corr, float grad_scale,
                                          int zero_grad) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gr = g[i] * grad_scale;
    float P = p[i] * decay;                                                     // decay == 1 when weight_decay == 0
    const float M = rn<TM>(fmaf(alpha1, gr, rn<TM>(st_load<TM>(m, i) * beta1)));  // add_(alpha) is a fused multiply-add
    const float V = rn<TV>(fmaf(__fmul_rn(alpha2, gr), gr, rn<TV>(st_load<TV>(v, i) * beta2)));   // addcmul contracts to an FMA
    const float cv = rn<TV>(rn<TV>(rn<TV>(sqrtf(V)) / denom_corr) + eps);
    const float upd = __fdiv_rn(__fmul_rn(neg_step_size, M), cv);               // addcdiv: (value * t1) / t2
    if (KAHAN) {
      float C = rn<TC>(__fadd_rn(st_load<TC>(comp, i), upd));
      const float T = P;
      P = __fadd_rn(P, C);
      C = rn<TC>(__fadd_rn(C, __fsub_rn(T, P)));
      st_store<TC>(comp, i, C);
    } else {
      P = __fadd_rn(P, upd);
    }
    p[i] = P;
    st_store<TM>(m, i, M);
    st_store<TV>(v, i, V);
    if (zero_grad) g[i] = 0.f;
    if (p_bf16) p_bf16[i] = __float2bfloat16_rn(P);
  }
}


// Standalone activation (the encoders fuse it into the FC1 GEMM epilogue; this serves `SiLU()(x)` / `nn.GELU` called
// on their own): y = x * sigmoid(1.702 x) (activation.py:24-25) or exact-erf GELU, fp32 in / out.
__global__ void act_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, int kind) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = x[i];
    y[i] = kind == ACT_QUICK_GELU ? v / (1.f + __expf(-1.702f * v)) : 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
  }
}
// nn.ReLU() called on its own, exact: a kernel of its own so that the GELU kinds' kernel stays as it is
__global__ void relu_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = fmaxf(x[i], 0.f);
}

}  // namespace mmb

using namespace mmb;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define LAUNCH_RC() ((int)cudaGetLastError())

extern "C" int mmb_cast_f32_to_bf16(const float* src, void* dst, long long n, void* stream) {
  if (n <= 0) return MMB_OK;
  if ((reinterpret_cast<uintptr_t>(src) & 15) || (reinterpret_cast<uintptr_t>(dst) & 7)) return MMB_ERR_ARG;
  cast_f32_bf16_kernel<false><<<grid_for(n / 4 + 1, 256), 256, 0, ST(stream)>>>(src, (__nv_bfloat16*)dst, n,
                                                                                 nullptr, 0);
  return LAUNCH_RC();
}

extern "C" int mmb_cast_f32_to_bf16_scaled(const float* src, void* dst, long long n, const float* scale,
                                           long long per_scale, void* stream) {
  if (n <= 0) return MMB_OK;
  if ((reinterpret_cast<uintptr_t>(src) & 15) || (reinterpret_cast<uintptr_t>(dst) & 7)) return MMB_ERR_ARG;
  if (!scale || per_scale <= 0 || (per_scale & 3)) return MMB_ERR_ARG;
  cast_f32_bf16_kernel<true><<<grid_for(n / 4 + 1, 256), 256, 0, ST(stream)>>>(src, (__nv_bfloat16*)dst, n, scale,
                                                                                per_scale);
  return LAUNCH_RC();
}

extern "C" int mmb_cast_bf16_to_f32(const void* src, float* dst, long long n, void* stream) {
  if (n <= 0) return MMB_OK;
  if ((reinterpret_cast<uintptr_t>(dst) & 15) || (reinterpret_cast<uintptr_t>(src) & 7)) return MMB_ERR_ARG;
  cast_bf16_f32_kernel<<<grid_for(n / 4 + 1, 256), 256, 0, ST(stream)>>>((const __nv_bfloat16*)src, dst, n);
  return LAUNCH_RC();
}

extern "C" int mmb_im2col_patches(const float* img, void* out, long long ld_out, int B, int H, int W, int ps,
                                  void* stream) {
  if (B <= 0 || ps <= 0 || (ps & 1) || H % ps || W % ps || (ld_out & 1) || ld_out < 3LL * ps * ps) return MMB_ERR_ARG;
  const long long total2 = (long long)B * (H / ps) * (W / ps) * 3 * ps * ps / 2;
  im2col_kernel<<<grid_for(total2, 256), 256, 0, ST(stream)>>>(img, (__nv_bfloat16*)out, B, H, W, ps, ld_out);
  return LAUNCH_RC();
}

static inline bool ln_dim_ok(int d) { return d > 0 && (d & 127) == 0 && (d >> 7) <= LN_MAX_NV; }

extern "C" int mmb_add_layernorm_fwd(const float* x_in, const void* y_bf16, float* x_out, void* ln_bf16, float* ln_f32,
                                     const float* gamma, const float* beta, float* mean, float* rstd,
                                     const int* row_idx, int rows_per_group, int M, int d, float eps, void* stream) {
  if (!ln_dim_ok(d)) return MMB_ERR_UNSUPPORTED;
  if (M <= 0) return MMB_OK;
  add_ln_fwd_kernel<false><<<grid_for(M, 8), 256, 0, ST(stream)>>>(x_in, (const __nv_bfloat16*)y_bf16, x_out,
                                                                    (__nv_bfloat16*)ln_bf16, ln_f32, gamma, beta, mean,
                                                                    rstd, row_idx, rows_per_group, M, d, eps, nullptr, 0);
  return LAUNCH_RC();
}

extern "C" int mmb_add_layernorm_fwd_scaled(const float* x_in, const void* y_bf16, float* x_out, void* ln_bf16,
                                            float* ln_f32, const float* gamma, const float* beta, float* mean,
                                            float* rstd, const float* scale, int rows_per_scale, int M, int d,
                                            float eps, void* stream) {
  if (!ln_dim_ok(d)) return MMB_ERR_UNSUPPORTED;
  if (!y_bf16 || !scale || rows_per_scale <= 0) return MMB_ERR_ARG;
  if (M <= 0) return MMB_OK;
  add_ln_fwd_kernel<true><<<grid_for(M, 8), 256, 0, ST(stream)>>>(x_in, (const __nv_bfloat16*)y_bf16, x_out,
                                                                   (__nv_bfloat16*)ln_bf16, ln_f32, gamma, beta, mean,
                                                                   rstd, nullptr, 0, M, d, eps, scale, rows_per_scale);
  return LAUNCH_RC();
}

extern "C" int mmb_vit_embed_ln_fwd(const void* patch_out, const float* cls, const float* pos, const float* gamma,
                                    const float* beta, float* x0, float* mean, float* rstd, int B, int S, int d,
                                    float eps, void* stream) {
  if (!ln_dim_ok(d)) return MMB_ERR_UNSUPPORTED;
  vit_embed_ln_fwd_kernel<<<grid_for((long long)B * S, 8), 256, 0, ST(stream)>>>(
      (const __nv_bfloat16*)patch_out, cls, pos, gamma, beta, x0, mean, rstd, B, S, d, eps);
  return LAUNCH_RC();
}

extern "C" int mmb_layernorm_bwd(const float* x, const void* dy_bf16, const float* dy_f32, const float* mean,
                                 const float* rstd, const float* gamma, const float* g_in, float* g_out, void* g_bf16,
                                 float* dgamma, float* dbeta, const int* row_idx, int rows_per_group, int M, int d,
                                 float* gsum, void* stream) {
  if (!ln_dim_ok(d)) return MMB_ERR_UNSUPPORTED;
  if (M <= 0) return MMB_OK;
  if (gsum && !g_bf16) return MMB_ERR_ARG;
  LnBwdArgs a{};
  a.gsum = gsum;
  a.x = x; a.dy_bf16 = (const __nv_bfloat16*)dy_bf16; a.dy_f32 = dy_f32; a.mean = mean; a.rstd = rstd; a.gamma = gamma;
  a.g_in = g_in; a.g_out = g_out; a.g_bf16 = (__nv_bfloat16*)g_bf16; a.dgamma = dgamma; a.dbeta = dbeta;
  a.row_idx = row_idx; a.rows_per_group = rows_per_group; a.M = M; a.d = d;
  return launch_ln_bwd<false>(a, ST(stream));
}

extern "C" int mmb_layernorm_bwd_scaled(const float* x, const void* dy_bf16, const float* dy_f32, const float* mean,
                                        const float* rstd, const float* gamma, const float* g_in, float* g_out,
                                        void* g_bf16, float* dgamma, float* dbeta, const float* scale,
                                        int rows_per_scale, int M, int d, float* gsum, void* stream) {
  if (!ln_dim_ok(d)) return MMB_ERR_UNSUPPORTED;
  if (!g_bf16 || !scale || rows_per_scale <= 0) return MMB_ERR_ARG;
  if (M <= 0) return MMB_OK;
  LnBwdArgs a{};
  a.gsum = gsum;
  a.x = x; a.dy_bf16 = (const __nv_bfloat16*)dy_bf16; a.dy_f32 = dy_f32; a.mean = mean; a.rstd = rstd; a.gamma = gamma;
  a.g_in = g_in; a.g_out = g_out; a.g_bf16 = (__nv_bfloat16*)g_bf16; a.dgamma = dgamma; a.dbeta = dbeta;
  a.M = M; a.d = d; a.scale = scale; a.rows_per_scale = rows_per_scale;
  return launch_ln_bwd<false, true>(a, ST(stream));
}

extern "C" int mmb_vit_embed_ln_bwd(const void* patch_out, const float* cls, const float* pos, const float* dy_f32,
                                    const float* mean, const float* rstd, const float* gamma, float* dt_f32,
                                    void* dpatch_bf16, float* dgamma, float* dbeta, int B, int S, int d,
                                    void* stream) {
  if (!ln_dim_ok(d)) return MMB_ERR_UNSUPPORTED;
  LnBwdArgs a{};
  a.patch_out = (const __nv_bfloat16*)patch_out; a.cls = cls; a.pos = pos; a.S = S;
  a.dy_f32 = dy_f32; a.mean = mean; a.rstd = rstd; a.gamma = gamma; a.g_out = dt_f32;
  a.g_bf16 = (__nv_bfloat16*)dpatch_bf16;
  a.dgamma = dgamma; a.dbeta = dbeta; a.M = B * S; a.d = d;
  return launch_ln_bwd<true>(a, ST(stream));
}

extern "C" int mmb_batch_sum(const float* in, float* out, int Bn, long long ld, int n, void* stream) {
  if (n & 3) return MMB_ERR_ARG;
  if (n <= 0 || Bn <= 0) return MMB_OK;   // empty sum: out is unchanged (the chunking below divides by both)
  const int bx = (n / 4 + 127) / 128;
  int chunks = (num_sms() * 4 + bx - 1) / bx;
  if (chunks > Bn) chunks = Bn;
  if (chunks < 1) chunks = 1;
  const int b_chunk = (Bn + chunks - 1) / chunks;
  dim3 grid(bx, (Bn + b_chunk - 1) / b_chunk);
  float* part = static_cast<float*>(scratch(SCR_BATCH_SUM, (size_t)grid.y * n * sizeof(float), ST(stream)));
  if (!part) return (int)cudaErrorMemoryAllocation;
  batch_sum_kernel<<<grid, 128, 0, ST(stream)>>>(in, part, Bn, ld, n, b_chunk);
  const int rc = LAUNCH_RC();
  return rc ? rc : reduce_partials(part, (int)grid.y, n, n, out, 1, ST(stream));
}

extern "C" int mmb_colsum_bf16(const void* x, float* out, int M, int N, long long ld, void* stream) {
  if ((N & 7) || (ld & 7)) return MMB_ERR_ARG;
  if (M <= 0 || N <= 0) return MMB_OK;   // empty sum: out is unchanged (the chunking below divides by both)
  const int bx = (N + 255) / 256;
  int chunks = (num_sms() * 6 + bx - 1) / bx;
  int rows_per_block = (M + chunks - 1) / chunks;
  rows_per_block = ((rows_per_block + 7) / 8) * 8;
  dim3 grid(bx, (M + rows_per_block - 1) / rows_per_block);
  float* part = static_cast<float*>(scratch(SCR_COLSUM, (size_t)grid.y * N * sizeof(float), ST(stream)));
  if (!part) return (int)cudaErrorMemoryAllocation;
  colsum_bf16_kernel<<<grid, 256, 0, ST(stream)>>>((const __nv_bfloat16*)x, part, M, N, ld, rows_per_block);
  const int rc = LAUNCH_RC();
  return rc ? rc : reduce_partials(part, (int)grid.y, N, N, out, 1, ST(stream));
}

extern "C" int mmb_text_embed_fwd(const long long* tokens, const float* emb, const float* pos, float* x, int B, int S,
                                  int d, int V, void* stream) {
  if (d & 3) return MMB_ERR_ARG;
  text_embed_fwd_kernel<<<grid_for((long long)B * S * d / 4, 256), 256, 0, ST(stream)>>>(tokens, emb, pos, x, B, S, d, V);
  return LAUNCH_RC();
}
extern "C" int mmb_text_embed_bwd(const long long* tokens, const float* g, float* demb, int B, int S, int d,
                                  void* stream) {
  if (d & 3) return MMB_ERR_ARG;
  text_embed_bwd_kernel<<<num_sms() * 4, 256, 0, ST(stream)>>>(tokens, g, demb, B * S, d);
  return LAUNCH_RC();
}
extern "C" int mmb_argmax_tokens(const long long* tokens, int* idx, int B, int S, void* stream) {
  argmax_tokens_kernel<<<(B + 7) / 8, 256, 0, ST(stream)>>>(tokens, idx, B, S);
  return LAUNCH_RC();
}
extern "C" int mmb_l2norm_fwd(const float* x, float* y, void* y_bf16, float* inv_norm, int B, int E, float eps,
                              void* stream) {
  l2norm_fwd_kernel<<<(B + 7) / 8, 256, 0, ST(stream)>>>(x, y, (__nv_bfloat16*)y_bf16, inv_norm, B, E, eps);
  return LAUNCH_RC();
}
extern "C" int mmb_l2norm_bwd(const float* dy, const float* y, const float* inv_norm, float* dx, void* dx_bf16, int B,
                              int E, void* stream) {
  l2norm_bwd_kernel<<<(B + 7) / 8, 256, 0, ST(stream)>>>(dy, y, inv_norm, dx, (__nv_bfloat16*)dx_bf16, B, E);
  return LAUNCH_RC();
}
extern "C" int mmb_adamw_step(float* p, float* g, float* m, float* v, void* p_bf16, long long n, float lr, float beta1,
                              float beta2, float eps, float weight_decay, int step, float grad_scale, int zero_grad,
                              void* stream) {
  if (n & 3) return MMB_ERR_ARG;
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  adamw_kernel<<<grid_for(n / 4, 256), 256, 0, ST(stream)>>>(p, g, m, v, (__nv_bfloat16*)p_bf16, n, lr, beta1, beta2,
                                                              eps, weight_decay, bc1, bc2, grad_scale, zero_grad);
  return LAUNCH_RC();
}
extern "C" int mmb_memset_async(void* p, int value, long long bytes, void* stream) {
  return (int)cudaMemsetAsync(p, value, (size_t)bytes, ST(stream));
}

extern "C" int mmb_bert_embed_ln_fwd(const long long* ids, const long long* type_ids, const float* word, const float* pos,
                                     const float* type, const float* gamma, const float* beta, float* x,
                                     unsigned char* kmask_out, long long pad_id, int B, int S, int d, int V, float eps,
                                     void* stream) {
  if (!ln_dim_ok(d)) return MMB_ERR_UNSUPPORTED;
  bert_embed_ln_fwd_kernel<<<grid_for((long long)B * S, 8), 256, 0, ST(stream)>>>(ids, type_ids, word, pos, type, gamma,
                                                                                 beta, x, kmask_out, pad_id, B, S, d, V,
                                                                                 eps);
  return LAUNCH_RC();
}
extern "C" int mmb_vit_assemble_fwd(const void* patch_out, const float* cls, const float* pos, const float* mask_token,
                                    const unsigned char* patch_mask, float* x, int B, int S, int d, void* stream) {
  if (d & 3) return MMB_ERR_ARG;
  vit_assemble_fwd_kernel<<<grid_for((long long)B * S * d / 4, 256), 256, 0, ST(stream)>>>(
      (const __nv_bfloat16*)patch_out, cls, pos, mask_token, patch_mask, x, B, S, d);
  return LAUNCH_RC();
}
extern "C" int mmb_coca_text_embed_fwd(const long long* ids, const float* emb, const float* cls, const float* pos,
                                       float* x, int B, int S, int d, int V, void* stream) {
  if (d & 3) return MMB_ERR_ARG;
  coca_text_embed_fwd_kernel<<<grid_for((long long)B * S * d / 4, 256), 256, 0, ST(stream)>>>(ids, emb, cls, pos, x, B, S,
                                                                                              d, V);
  return LAUNCH_RC();
}
extern "C" int mmb_ce_labels(const float* logits, long long ld, const long long* labels, long long label_stride,
                             long long ignore_index, int M, int V, float* row_loss, float* accum, void* stream) {
  if (M <= 0 || V <= 0 || !accum) return MMB_ERR_ARG;
  float* part2 = static_cast<float*>(scratch(SCR_LOSS, 2ull * M * sizeof(float), ST(stream)));
  if (!part2) return (int)cudaErrorMemoryAllocation;
  ce_labels_kernel<<<M, 256, 0, ST(stream)>>>(logits, ld, labels, label_stride, ignore_index, M, V, row_loss, part2);
  const int rc = LAUNCH_RC();
  return rc ? rc : reduce_partials(part2, M, 2, 2, accum, 1, ST(stream));
}
extern "C" int mmb_gather_rows_cast(const float* x, void* out_bf16, int B, int rows_per_group, int row, int d,
                                    void* stream) {
  if (d & 3) return MMB_ERR_ARG;
  gather_rows_cast_kernel<<<grid_for((long long)B * d / 4, 256), 256, 0, ST(stream)>>>(x, (__nv_bfloat16*)out_bf16, B,
                                                                                     rows_per_group, row, d);
  return LAUNCH_RC();
}
extern "C" int mmb_gather_rows_idx_cast(const float* x, long long ld, const long long* idx, void* out_bf16, int n, int d,
                                        void* stream) {
  if ((d & 3) || (ld & 3) || n < 0) return MMB_ERR_ARG;
  if (n == 0) return MMB_OK;
  gather_rows_idx_cast_kernel<<<grid_for((long long)n * d / 4, 256), 256, 0, ST(stream)>>>(x, ld, idx,
                                                                                           (__nv_bfloat16*)out_bf16, n, d);
  return LAUNCH_RC();
}
extern "C" int mmb_tanh_inplace(float* x, long long n, void* stream) {
  tanh_inplace_kernel<<<grid_for(n, 256), 256, 0, ST(stream)>>>(x, n);
  return LAUNCH_RC();
}
extern "C" int mmb_concat_tokens(const float* cls, const float* a, const float* b, float* out, int B, int Sa, int Sb,
                                 int d, void* stream) {
  if (d & 3) return MMB_ERR_ARG;
  const long long total = (long long)B * ((cls ? 1 : 0) + Sa + Sb) * d / 4;
  concat_tokens_kernel<<<grid_for(total, 256), 256, 0, ST(stream)>>>(cls, a, b, out, B, Sa, Sb, d);
  return LAUNCH_RC();
}

// dtype codes: 0 = fp32, 1 = bf16.  Hyper-parameters arrive as doubles (Python floats) and are folded / rounded to
// fp32 exactly where the reference does: 1 - lr*wd and 1 - beta are formed in double, then cast.
extern "C" int mmb_anyprecision_adamw_step(float* p, float* g, void* m, int m_dtype, void* v, int v_dtype, void* comp,
                                           int comp_dtype, void* p_bf16, long long n, double lr, double beta1,
                                           double beta2, double eps, double weight_decay, int step, float grad_scale,
                                           int zero_grad, void* stream) {
  if (n <= 0) return MMB_OK;
  if (!p || !g || !m || !v || step < 1) return MMB_ERR_ARG;
  if ((m_dtype | v_dtype | comp_dtype) & ~1) return MMB_ERR_ARG;
  // bias corrections as the reference computes them on a float32 step tensor (anyprecision.py:167-172)
  const float b1f = (float)beta1, b2f = (float)beta2;
  const float bc1 = 1.f - powf(b1f, (float)step);
  const float neg_step_size = -((1.f / bc1) * (float)lr);   // `lr / tensor` is reciprocal(tensor) * lr in torch (Tensor.__rtruediv__)
  const float denom_corr = sqrtf(1.f - powf(b2f, (float)step));
  const float decay = weight_decay != 0.0 ? (float)(1.0 - lr * weight_decay) : 1.f;
  const float alpha1 = (float)(1.0 - beta1), alpha2 = (float)(1.0 - beta2);
  const int grid = grid_for(n, 256);
  typedef __nv_bfloat16 bf;
#define AP_LAUNCH(TM, TV, TC, K)                                                                                      \
  anyprecision_adamw_kernel<TM, TV, TC, K><<<grid, 256, 0, ST(stream)>>>(p, g, (TM*)m, (TV*)v, (TC*)comp, (bf*)p_bf16, n, \
                                                                         decay, b1f, b2f, alpha1, alpha2, (float)eps,  \
                                                                         neg_step_size, denom_corr, grad_scale, zero_grad)
#define AP_COMP(TM, TV)                                                                   \
  do {                                                                                    \
    if (!comp) AP_LAUNCH(TM, TV, float, false);                                           \
    else if (comp_dtype == 0) AP_LAUNCH(TM, TV, float, true);                             \
    else AP_LAUNCH(TM, TV, bf, true);                                                     \
  } while (0)
  if (m_dtype == 0 && v_dtype == 0) AP_COMP(float, float);
  else if (m_dtype == 0 && v_dtype == 1) AP_COMP(float, bf);
  else if (m_dtype == 1 && v_dtype == 0) AP_COMP(bf, float);
  else AP_COMP(bf, bf);
#undef AP_COMP
#undef AP_LAUNCH
  return LAUNCH_RC();
}

extern "C" int mmb_act_fwd(const float* x, float* y, long long n, int kind, void* stream) {
  if (n <= 0) return MMB_OK;
  if (kind == ACT_RELU) relu_fwd_kernel<<<grid_for(n, 256), 256, 0, ST(stream)>>>(x, y, n);
  else if (kind == ACT_QUICK_GELU || kind == ACT_GELU_ERF) act_fwd_kernel<<<grid_for(n, 256), 256, 0, ST(stream)>>>(x, y, n, kind);
  else return MMB_ERR_ARG;
  return LAUNCH_RC();
}
