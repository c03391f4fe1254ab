// Temperature-scaled softmax cross-entropy over similarity rows: statistics pass + gradient pass.
// Restates modules/losses/contrastive_loss_with_temperature.py:81-107 for one direction (a->b or b->a):
//   logits = exp(logit_scale) * sims ; loss_i = CE(logits_i, label_i = label_offset + i) (+ label smoothing)
// and emits d(mean loss * loss_weight)/d sims in bf16 (operand of the embedding-gradient GEMMs) plus the
// contribution to d/d logit_scale (= sum dlogits * logits, because d logits / d logit_scale = logits).
#include "common.cuh"
#include "mmb200_internal.h"

namespace mmb {

__device__ __forceinline__ float block_reduce_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) r = fmaxf(r, red[i]);
  return r;
}
__device__ __forceinline__ float block_reduce_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) r += red[i];
  return r;
}

// Pass 1 (per local row i): logits = T * sims; row LSE; loss_i (with label smoothing); optional logits output;
// row i's share of d loss / d logit_scale written to dscale_part[i] (summed in row order by the host wrapper).
// label(i) = label_offset + i.
__global__ void contrastive_ce_stats_kernel(const float* __restrict__ sims, long long ld,
                                            const float* __restrict__ logit_scale, int rows, int N, int label_offset,
                                            float smoothing, float loss_weight, float* __restrict__ row_loss,
                                            float* __restrict__ lse_out, float* __restrict__ dscale_part,
                                            float* __restrict__ logits_out, long long ld_l,
                                            const float* __restrict__ row_w) {
  __shared__ float red[32];
  const int i = blockIdx.x;
  if (i >= rows) return;
  const float T = __expf(*logit_scale);
  const float* srow = sims + (long long)i * ld;
  const int label = label_offset + i;
  float mx = -INFINITY, sm = 0.f;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    const float l = T * srow[j];
    mx = fmaxf(mx, l);
    sm += l;
    if (logits_out) logits_out[(long long)i * ld_l + j] = l;
  }
  mx = block_reduce_max(mx, red);
  const float mean_logit = block_reduce_sum(sm, red) / N;
  float se = 0.f;
  for (int j = threadIdx.x; j < N; j += blockDim.x) se += __expf(T * srow[j] - mx);
  se = block_reduce_sum(se, red);
  const float lse = mx + logf(se);
  const float l_label = T * srow[label];
  const float loss = (1.f - smoothing) * (lse - l_label) + smoothing * (lse - mean_logit);
  // row_w (optional): per-row weight of the mean, mask_i / count(mask) (contrastive_loss_with_temperature.py:97-100
  // selects rows before F.cross_entropy(reduction="mean")); without it every row weighs 1 / rows.
  const float wrow = row_w ? row_w[i] : 1.f / rows;
  if (threadIdx.x == 0) {
    if (row_loss) row_loss[i] = row_w ? loss * wrow * rows : loss;  // so that sum(row_loss) / rows is the masked mean
    if (lse_out) lse_out[i] = lse;
  }
  if (dscale_part) {
    // d loss_i / d logit_scale = sum_j (p_ij - (1-eps) y_ij - eps/N) * logit_ij   (d logit / d logit_scale = logit)
    float acc = 0.f;
    for (int j = threadIdx.x; j < N; j += blockDim.x) {
      const float l = T * srow[j];
      float gl = __expf(l - lse) - smoothing / N;
      if (j == label) gl -= (1.f - smoothing);
      acc += gl * l;
    }
    acc = block_reduce_sum(acc, red);
    if (threadIdx.x == 0) dscale_part[i] = acc * loss_weight * wrow;
  }
}

// Pass 2: gradient w.r.t. the similarity row-block of THIS rank, including (columns [col_lo, col_hi)) the part that
// the reference obtains by reduce-scattering the gradient of the all-gathered embeddings:
//   dsims[i,j] = gs*T*[ softmax_row(L)[i,j] - t_ij ]  +  1[col_lo<=j<col_hi] * gs*T*[ exp(L[i,j] - lse_col[j]) - t_ij ]
// with t_ij = (1-eps)*1[j==label(i)] + eps/N and lse_col[j] the row-LSE of the OTHER direction's global row j
// (L_other[j, i] == L[i, j]).  GLOBAL backprop: whole range; LOCAL: own block; NONE: empty range.
__global__ void contrastive_ce_grad_kernel(const float* __restrict__ sims, long long ld,
                                           const float* __restrict__ logit_scale, int rows, int N, int label_offset,
                                           float smoothing, float loss_weight, const float* __restrict__ lse_row,
                                           const float* __restrict__ lse_col, int col_lo, int col_hi,
                                           __nv_bfloat16* __restrict__ dsims, float* __restrict__ dsims_f32,
                                           long long ld_d, const float* __restrict__ row_w,
                                           const float* __restrict__ col_w) {
  const int i = blockIdx.x;
  if (i >= rows) return;
  const float T = __expf(*logit_scale);
  const float* srow = sims + (long long)i * ld;
  const int label = label_offset + i;
  const float lse = lse_row[i];
  // row weights: this rank's masked-mean weights; col_w[j]: the weight global row j carries in ITS rank's mean
  const float gsT = loss_weight * T * (row_w ? row_w[i] : 1.f / rows);
  const float gcT = loss_weight * T / rows;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    const float l = T * srow[j];
    const float t = ((j == label) ? (1.f - smoothing) : 0.f) + smoothing / N;
    float g = gsT * (__expf(l - lse) - t);
    if (lse_col && j >= col_lo && j < col_hi) {
      const float wc = col_w ? loss_weight * T * col_w[j] : gcT;
      if (wc != 0.f) g += wc * (__expf(l - lse_col[j]) - t);  // masked-out peer rows may carry a non-finite LSE
    }
    if (dsims) dsims[(long long)i * ld_d + j] = __float2bfloat16(g);
    if (dsims_f32) dsims_f32[(long long)i * ld_d + j] = g;
  }
}

// Combines the per-(row, 128-column part) online-softmax statistics written by the fused similarity GEMM
// (gemm.cu, EPI_CE_STATS: float4 {max, sum e^(x-max), sum e^(x-max) x, sum x}, x = T * sim) into what
// contrastive_ce_stats_kernel derives from materialised logits: row LSE, row loss (label smoothing, row weights) and
// the contribution to d loss / d logit_scale = sum_j (p_ij - t_ij) x_ij = E_p[x] - (1-eps) x_label - eps mean(x).
// One warp per row; parts with an empty column range carry sum == 0 and are skipped.
__global__ void ce_stats_reduce_kernel(const float4* __restrict__ part, int part_ld, int n_parts,
                                       const float* __restrict__ xlabel, int rows, int n_total, float smoothing,
                                       float loss_weight, const float* __restrict__ row_w, float* __restrict__ row_loss,
                                       float* __restrict__ lse_out, float* __restrict__ dscale_part) {
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= rows) return;
  const float4* pr = part + (long long)i * part_ld;
  float mx = -INFINITY;
  for (int k = lane; k < n_parts; k += 32) {
    const float4 q = pr[k];
    if (q.y > 0.f) mx = fmaxf(mx, q.x);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float se = 0.f, sex = 0.f, sx = 0.f;
  for (int k = lane; k < n_parts; k += 32) {
    const float4 q = pr[k];
    if (q.y > 0.f) {
      const float w = __expf(q.x - mx);
      se += q.y * w; sex += q.z * w;
    }
    sx += q.w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    se += __shfl_xor_sync(0xffffffffu, se, o);
    sex += __shfl_xor_sync(0xffffffffu, sex, o);
    sx += __shfl_xor_sync(0xffffffffu, sx, o);
  }
  if (lane == 0) {
    const float lse = mx + logf(se);
    const float l_label = xlabel[i];
    const float mean_logit = sx / n_total;
    const float loss = (1.f - smoothing) * (lse - l_label) + smoothing * (lse - mean_logit);
    const float wrow = row_w ? row_w[i] : 1.f / rows;
    if (row_loss) row_loss[i] = row_w ? loss * wrow * rows : loss;
    if (lse_out) lse_out[i] = lse;
    if (dscale_part)
      dscale_part[i] = (sex / se - (1.f - smoothing) * l_label - smoothing * mean_logit) * loss_weight * wrow;
  }
}

// Label cross-entropy from the fused GEMM's partial statistics (Linear -> nn.CrossEntropyLoss(ignore_index) heads,
// models/coca/coca_model.py:447-452): accum[0] += sum over kept rows of (lse - x_label), accum[1] += number of kept rows.
__global__ void ce_labels_reduce_kernel(const float4* __restrict__ part, int part_ld, int n_parts,
                                        const float* __restrict__ xlabel, const int* __restrict__ labels, int ignore_index,
                                        int rows, float* __restrict__ row_loss, float* __restrict__ part2) {
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= rows) return;
  if (labels[i] == ignore_index) {
    if (lane == 0) {
      if (row_loss) row_loss[i] = 0.f;
      part2[2 * i] = 0.f; part2[2 * i + 1] = 0.f;
    }
    return;
  }
  const float4* pr = part + (long long)i * part_ld;
  float mx = -INFINITY;
  for (int k = lane; k < n_parts; k += 32) {
    const float4 q = pr[k];
    if (q.y > 0.f) mx = fmaxf(mx, q.x);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float se = 0.f;
  for (int k = lane; k < n_parts; k += 32) {
    const float4 q = pr[k];
    if (q.y > 0.f) se += q.y * __expf(q.x - mx);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
  if (lane == 0) {
    const float loss = mx + logf(se) - xlabel[i];
    if (row_loss) row_loss[i] = loss;
    part2[2 * i] = loss; part2[2 * i + 1] = 1.f;
  }
}

// out[0] = scale * sum(in[0..n))  (deterministic single-block tree; n is a batch size)
__global__ void sum_scale_kernel(const float* __restrict__ in, int n, float scale, float* __restrict__ out, int accumulate) {
  __shared__ float red[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += in[i];
  s = block_reduce_sum(s, red);
  if (threadIdx.x == 0) out[0] = (accumulate ? out[0] : 0.f) + s * scale;
}


// Plain fp32 SIMT matmul for the tiny / unaligned shapes the tensor-core path rejects (e.g. the reference's own
// 3x5 known-answer tests).  C[M,N] (+)= alpha * op(A) op(B);  ta: A stored [K,M];  tb: B stored [N,K].
__global__ void matmul_f32_kernel(const float* __restrict__ A, long long lda, int ta, const float* __restrict__ B,
                                  long long ldb, int tb, float* __restrict__ C, long long ldc, int M, int N, int K,
                                  float alpha, int accumulate) {
  __shared__ float sa[32][33], sb[32][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int row = blockIdx.y * 32 + ty, col = blockIdx.x * 32 + tx;
  float acc = 0.f;
  for (int k0 = 0; k0 < K; k0 += 32) {
    {  // sa[m][k]
      const int m = blockIdx.y * 32 + ty, k = k0 + tx;
      float v = 0.f;
      if (m < M && k < K) v = ta ? A[(long long)k * lda + m] : A[(long long)m * lda + k];
      sa[ty][tx] = v;
    }
    {  // sb[k][n]
      const int k = k0 + ty, n = blockIdx.x * 32 + tx;
      float v = 0.f;
      if (k < K && n < N) v = tb ? B[(long long)n * ldb + k] : B[(long long)k * ldb + n];
      sb[ty][tx] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 32; ++k) acc += sa[ty][k] * sb[k][tx];
    __syncthreads();
  }
  if (row < M && col < N) {
    float* c = C + (long long)row * ldc + col;
    *c = (accumulate ? *c : 0.f) + alpha * acc;
  }
}

}  // namespace mmb

using namespace mmb;

extern "C" int mmb_contrastive_ce_stats(const float* sims, long long ld, const float* logit_scale, int rows, int N,
                                        int label_offset, float label_smoothing, float loss_weight, float* row_loss,
                                        float* lse_out, float* dscale_accum, float* logits_out, long long ld_l,
                                        const float* row_w, void* stream) {
  if (rows <= 0 || N <= 0 || label_offset < 0 || label_offset + rows > N) return MMB_ERR_ARG;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* dpart = nullptr;
  if (dscale_accum && !(dpart = static_cast<float*>(scratch(SCR_LOSS, (size_t)rows * sizeof(float), st))))
    return (int)cudaErrorMemoryAllocation;
  contrastive_ce_stats_kernel<<<rows, 256, 0, st>>>(sims, ld, logit_scale, rows, N, label_offset, label_smoothing,
                                                    loss_weight, row_loss, lse_out, dpart, logits_out, ld_l, row_w);
  const int rc = (int)cudaGetLastError();
  return (rc || !dscale_accum) ? rc : reduce_partials(dpart, rows, 1, 1, dscale_accum, 1, st);
}

extern "C" int mmb_contrastive_ce_grad(const float* sims, long long ld, const float* logit_scale, int rows, int N,
                                       int label_offset, float label_smoothing, float loss_weight,
                                       const float* lse_row, const float* lse_col, int col_lo, int col_hi,
                                       void* dsims_bf16, float* dsims_f32, long long ld_d, const float* row_w,
                                       const float* col_w, void* stream) {
  if (rows <= 0 || N <= 0 || label_offset < 0 || label_offset + rows > N || !lse_row) return MMB_ERR_ARG;
  contrastive_ce_grad_kernel<<<rows, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      sims, ld, logit_scale, rows, N, label_offset, label_smoothing, loss_weight, lse_row, lse_col, col_lo, col_hi,
      (__nv_bfloat16*)dsims_bf16, dsims_f32, ld_d, row_w, col_w);
  return (int)cudaGetLastError();
}

extern "C" int mmb_sum_scale(const float* in, int n, float scale, float* out, int accumulate, void* stream) {
  sum_scale_kernel<<<1, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(in, n, scale, out, accumulate);
  return (int)cudaGetLastError();
}

extern "C" int mmb_matmul_f32(const float* A, long long lda, int ta, const float* B, long long ldb, int tb, float* C,
                              long long ldc, int M, int N, int K, float alpha, int accumulate, void* stream) {
  if (M <= 0 || N <= 0 || K <= 0) return MMB_ERR_ARG;
  dim3 grid((N + 31) / 32, (M + 31) / 32), block(32, 32);
  matmul_f32_kernel<<<grid, block, 0, reinterpret_cast<cudaStream_t>(stream)>>>(A, lda, ta, B, ldb, tb, C, ldc, M, N, K,
                                                                               alpha, accumulate);
  return (int)cudaGetLastError();
}

extern "C" int mmb_ce_stats_reduce(const void* part, int part_ld, int n_parts, const float* xlabel, int rows, int n_total,
                                   float label_smoothing, float loss_weight, const float* row_w, float* row_loss,
                                   float* lse_out, float* dscale_accum, void* stream) {
  if (!part || !xlabel || rows <= 0 || n_parts <= 0 || n_parts > part_ld || n_total <= 0) return MMB_ERR_ARG;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* dpart = nullptr;
  if (dscale_accum && !(dpart = static_cast<float*>(scratch(SCR_LOSS, (size_t)rows * sizeof(float), st))))
    return (int)cudaErrorMemoryAllocation;
  ce_stats_reduce_kernel<<<(rows + 7) / 8, 256, 0, st>>>(reinterpret_cast<const float4*>(part), part_ld, n_parts, xlabel,
                                                         rows, n_total, label_smoothing, loss_weight, row_w, row_loss,
                                                         lse_out, dpart);
  const int rc = (int)cudaGetLastError();
  return (rc || !dscale_accum) ? rc : reduce_partials(dpart, rows, 1, 1, dscale_accum, 1, st);
}

extern "C" int mmb_ce_labels_reduce(const void* part, int part_ld, int n_parts, const float* xlabel, const int* labels,
                                    int ignore_index, int rows, float* row_loss, float* accum, void* stream) {
  if (!part || !xlabel || !labels || !accum || rows <= 0 || n_parts <= 0 || n_parts > part_ld) return MMB_ERR_ARG;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* part2 = static_cast<float*>(scratch(SCR_LOSS, 2ull * rows * sizeof(float), st));
  if (!part2) return (int)cudaErrorMemoryAllocation;
  ce_labels_reduce_kernel<<<(rows + 7) / 8, 256, 0, st>>>(reinterpret_cast<const float4*>(part), part_ld, n_parts, xlabel,
                                                          labels, ignore_index, rows, row_loss, part2);
  const int rc = (int)cudaGetLastError();
  return rc ? rc : reduce_partials(part2, rows, 2, 2, accum, 1, st);
}
