// Random patch dropping (FLIP, arXiv 2212.00794) on the ViT patch front end: PatchEmbeddings(patch_drop_rate=...)
// keeps L of the P patches of each image, in the order of a per-sample index keep[B, L] (int32, distinct entries per
// row).  The kernels here embed only the kept patches: im2col reads the kept patches' pixels and nothing else, so the
// conv GEMM and everything after it run on B*L rows.  Same conventions as elementwise.cu / embed_bwd.cu: 128-bit
// accesses along d, grid-stride loops, and no floating-point atomics (partials + a fixed-order reduction).
#include "common.cuh"
#include "mmb200_internal.h"

namespace mmb {

static inline int pd_grid(long long n_items, int per_block) {
  long long b = (n_items + per_block - 1) / per_block;
  const long long cap = (long long)num_sms() * 16;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

__device__ __forceinline__ int kept_patch(const int* __restrict__ keep, long long r, int P) {
  const int p = keep[r];
  if (p < 0 || p >= P) __trap();
  return p;
}

// im2col_kernel restricted to the kept patches: out row b*L+j holds patch keep[b,j] of image b, same K order
// (c, kh, kw) and row pitch.
__global__ void im2col_gather_kernel(const float* __restrict__ img, const int* __restrict__ keep,
                                     __nv_bfloat16* __restrict__ out, int B, int H, int W, int ps, int L,
                                     long long ld_out) {
  const int gp = W / ps, P = (H / ps) * gp, K = 3 * ps * ps;
  const long long total2 = (long long)B * L * K / 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total2;
       i += (long long)gridDim.x * blockDim.x) {
    const long long e = i * 2;
    const int k = (int)(e % K);
    const long long row = e / K;
    const int b = (int)(row / L);
    const int p = kept_patch(keep, row, P);
    const int c = k / (ps * ps), r = k % (ps * ps), kh = r / ps, kw = r % ps;
    const int py = p / gp, px = p % gp;
    const float2 v = __ldg(reinterpret_cast<const float2*>(
        img + (((long long)b * 3 + c) * H + (py * ps + kh)) * W + px * ps + kw));
    *reinterpret_cast<uint32_t*>(out + row * ld_out + k) = pack_bf16x2(v.x, v.y);
  }
}

// vit_assemble_fwd_kernel on the kept patches: x[b,0] = cls + pos[0] (with cls), and for j < L with p = keep[b,j]
//   x[b,off+j] = (mask[b,p] ? mask_token : patch_out[b*L+j]) + pos[off+p]
// (the mask flag belongs to the patch, so a kept patch keeps it).  One fp32 add per element, as the full kernel.
__global__ void vit_assemble_gather_fwd_kernel(const __nv_bfloat16* __restrict__ patch_out,
                                               const float* __restrict__ cls, const float* __restrict__ pos,
                                               const float* __restrict__ mask_token,
                                               const unsigned char* __restrict__ patch_mask,
                                               const int* __restrict__ keep, float* __restrict__ x, int B, int L, int P,
                                               int d) {
  const int d4 = d >> 2;
  const int off = cls ? 1 : 0, S = off + L;
  const long long total = (long long)B * S * d4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d4) * 4;
    const long long row = i / d4;
    const int s = (int)(row % S);
    const long long b = row / S;
    float4 a, t;
    if (s < off) {
      a = __ldg(reinterpret_cast<const float4*>(pos + c));
      t = __ldg(reinterpret_cast<const float4*>(cls + c));
    } else {
      const long long r = b * L + (s - off);
      const int p = kept_patch(keep, r, P);
      a = __ldg(reinterpret_cast<const float4*>(pos + (long long)(off + p) * d + c));
      if (patch_mask && mask_token && patch_mask[b * P + p]) {
        t = __ldg(reinterpret_cast<const float4*>(mask_token + c));
      } else {
        const uint2 u = *reinterpret_cast<const uint2*>(patch_out + r * d + c);
        t = make_float4(bf16_lo(u.x), bf16_hi(u.x), bf16_lo(u.y), bf16_hi(u.y));
      }
    }
    reinterpret_cast<float4*>(x)[i] = make_float4(a.x + t.x, a.y + t.y, a.z + t.z, a.w + t.w);
  }
}

// inv[b, p] = j where keep[b, j] = p, -1 for a dropped patch.  One CTA per sample.
__global__ void keep_inverse_kernel(const int* __restrict__ keep, int* __restrict__ inv, int L, int P) {
  const long long b = blockIdx.x;
  for (int p = threadIdx.x; p < P; p += blockDim.x) inv[b * P + p] = -1;
  __syncthreads();
  for (int j = threadIdx.x; j < L; j += blockDim.x) inv[b * P + kept_patch(keep, b * L + j, P)] = j;
}

// Patch rows of the backward: dpatch[b*L+j] = bf16(mask[b,keep[b,j]] ? 0 : g[b,off+j]).  With a mask, the thread
// also sums its strip's masked rows into mpart[strip] (dmask_token partials, added in strip order afterwards).
// One thread = one float4 column x a strip of `rows_per_strip` consecutive rows.
__global__ void __launch_bounds__(256) vit_assemble_gather_bwd_rows_kernel(
    const float* __restrict__ g, const unsigned char* __restrict__ patch_mask, const int* __restrict__ keep,
    __nv_bfloat16* __restrict__ dpatch, float* __restrict__ mpart, int B, int L, int P, int d, int off,
    int rows_per_strip) {
  const int d4 = d >> 2;
  const int S = off + L;
  const long long n_rows = (long long)B * L;
  const long long n_strips = (n_rows + rows_per_strip - 1) / rows_per_strip;
  const long long total = n_strips * d4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d4) * 4;
    const long long strip = i / d4;
    const long long r0 = strip * rows_per_strip;
    const long long r1 = r0 + rows_per_strip < n_rows ? r0 + rows_per_strip : n_rows;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    long long b = r0 / L;
    int j = (int)(r0 % L);
    for (long long r = r0; r < r1; ++r, ++j) {
      if (j == L) { j = 0; ++b; }
      const float4 v = *reinterpret_cast<const float4*>(g + (b * S + off + j) * d + c);
      const bool masked = patch_mask != nullptr && patch_mask[b * P + kept_patch(keep, r, P)] != 0;
      uint2 o = make_uint2(0u, 0u);
      if (masked) { acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; }
      else { o.x = pack_bf16x2(v.x, v.y); o.y = pack_bf16x2(v.z, v.w); }
      *reinterpret_cast<uint2*>(dpatch + r * d + c) = o;
    }
    if (mpart != nullptr) *reinterpret_cast<float4*>(mpart + strip * d + c) = acc;
  }
}

// Position-embedding rows of the backward, as batch_sum_kernel but gathered through the inverse map: for q < off
// (the CLS row) the chunk's sum of g[b,0]; for q = off+p the chunk's sum over the samples that kept p of
// g[b, off+inv[b,p]].  A patch no sample of the chunk kept sums to exactly 0.  part[blockIdx.y][(off+P)*d].
__global__ void patch_drop_pos_bwd_kernel(const float* __restrict__ g, const int* __restrict__ inv,
                                          float* __restrict__ part, int B, int L, int P, int d, int off, int b_chunk) {
  const int n = (off + P) * d;
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (e >= n) return;
  const int q = e / d, c = e % d;
  const long long S = off + L;
  const int b0 = blockIdx.y * b_chunk, b1 = min(b0 + b_chunk, B);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int b = b0; b < b1; ++b) {
    long long row;
    if (q < off) {
      row = (long long)b * S;
    } else {
      const int j = inv[(long long)b * P + (q - off)];
      if (j < 0) continue;
      row = (long long)b * S + off + j;
    }
    const float4 v = *reinterpret_cast<const float4*>(g + row * d + c);
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  *reinterpret_cast<float4*>(part + (long long)blockIdx.y * n + e) = acc;
}

}  // namespace mmb

using namespace mmb;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define LAUNCH_RC() ((int)cudaGetLastError())

extern "C" int mmb_im2col_patches_gather(const float* img, const int* keep, void* out, long long ld_out, int B, int H,
                                         int W, int ps, int L, void* stream) {
  if (B <= 0 || L <= 0 || ps <= 0 || (ps & 1) || H % ps || W % ps || (ld_out & 1) || ld_out < 3LL * ps * ps)
    return MMB_ERR_ARG;
  if (L > (H / ps) * (W / ps)) return MMB_ERR_ARG;
  const long long total2 = (long long)B * L * 3 * ps * ps / 2;
  im2col_gather_kernel<<<pd_grid(total2, 256), 256, 0, ST(stream)>>>(img, keep, (__nv_bfloat16*)out, B, H, W, ps, L,
                                                                      ld_out);
  return LAUNCH_RC();
}

extern "C" int mmb_vit_assemble_gather_fwd(const void* patch_out, const float* cls, const float* pos,
                                           const float* mask_token, const unsigned char* patch_mask, const int* keep,
                                           float* x, int B, int L, int P, int d, void* stream) {
  if ((d & 3) || B <= 0 || L <= 0 || L > P) return MMB_ERR_ARG;
  const long long S = L + (cls ? 1 : 0);
  vit_assemble_gather_fwd_kernel<<<pd_grid((long long)B * S * d / 4, 256), 256, 0, ST(stream)>>>(
      (const __nv_bfloat16*)patch_out, cls, pos, mask_token, patch_mask, keep, x, B, L, P, d);
  return LAUNCH_RC();
}

extern "C" int mmb_vit_assemble_gather_bwd(const float* g, const unsigned char* patch_mask, const int* keep,
                                           void* dpatch, float* dmask_token, float* dcls, float* dpos, int B, int L,
                                           int P, int d, int has_cls, void* stream) {
  if ((d & 3) || B <= 0 || L <= 0 || L > P || (dcls && !has_cls)) return MMB_ERR_ARG;
  const int off = has_cls ? 1 : 0;
  cudaStream_t st = ST(stream);
  // scratch: inverse map int32 [B, P] | position partials fp32 [chunks, (off+P)*d] | mask partials fp32 [strips, d]
  const int rows_per_strip = 32;
  const long long strips = ((long long)B * L + rows_per_strip - 1) / rows_per_strip;
  const int n = (off + P) * d;
  const int bx = (n / 4 + 127) / 128;
  int chunks = (num_sms() * 4 + bx - 1) / bx;
  if (chunks > B) chunks = B;
  if (chunks < 1) chunks = 1;
  const int b_chunk = (B + chunks - 1) / chunks;
  chunks = (B + b_chunk - 1) / b_chunk;
  const bool want_pos = dpos != nullptr || dcls != nullptr;
  const bool want_mask = dmask_token != nullptr && patch_mask != nullptr;
  const size_t inv_bytes = ((size_t)B * P * sizeof(int) + 255) & ~(size_t)255;
  const size_t pos_bytes = want_pos ? (((size_t)chunks * n * sizeof(float) + 255) & ~(size_t)255) : 0;
  const size_t mask_bytes = want_mask ? (size_t)strips * d * sizeof(float) : 0;
  char* scr = static_cast<char*>(scratch(SCR_PATCH_DROP, inv_bytes + pos_bytes + mask_bytes, st));
  if (!scr) return (int)cudaErrorMemoryAllocation;
  int* inv = reinterpret_cast<int*>(scr);
  float* ppart = reinterpret_cast<float*>(scr + inv_bytes);
  float* mpart = want_mask ? reinterpret_cast<float*>(scr + inv_bytes + pos_bytes) : nullptr;

  vit_assemble_gather_bwd_rows_kernel<<<pd_grid(strips * (d / 4), 256), 256, 0, st>>>(
      g, patch_mask, keep, (__nv_bfloat16*)dpatch, mpart, B, L, P, d, off, rows_per_strip);
  int rc = LAUNCH_RC();
  if (!rc && want_mask) rc = reduce_partials(mpart, (int)strips, d, d, dmask_token, 1, st);
  if (!rc && want_pos) {
    keep_inverse_kernel<<<B, 256, 0, st>>>(keep, inv, L, P);
    rc = LAUNCH_RC();
    if (!rc) {
      patch_drop_pos_bwd_kernel<<<dim3(bx, chunks), 128, 0, st>>>(g, inv, ppart, B, L, P, d, off, b_chunk);
      rc = LAUNCH_RC();
    }
    if (!rc && dpos) rc = reduce_partials(ppart, chunks, n, n, dpos, 1, st);
    if (!rc && dcls) rc = reduce_partials(ppart, chunks, d, n, dcls, 1, st);
  }
  return rc;
}
