// General scaled-dot-product attention forward for the shapes the fused self-attention kernels do not cover:
// cross-attention (separate Q and K/V sources, Sq != Skv), head_dim 64 / 96 / 128, batch-shared queries (learned
// pooler queries), arbitrary boolean masks.  One CTA per (batch, head); K and V of the head stay in shared memory,
// each warp owns 16 query rows and runs an online-softmax sweep over 64-key blocks on warp-level tensor-core MMAs.
// Shapes whose head does not fit (generic_resident_fits() in attention_generic.cuh) go to the K / V-streamed kernels
// of attention_generic_stream.cu.
//
// Serves CoCa (SURVEY.md §8 a14): AttentionPooler / CascadedAttentionPooler (modules/layers/attention_pooler.py:16-101,
// head_dim 96 for ViT-L/14), the text decoder's [causal x padding] mask with its CLS row (models/coca/text_decoder.py
// :141-162) and the multimodal decoder's cross-attention (modules/layers/transformer.py:354-377), i.e. the
// F.scaled_dot_product_attention calls of modules/layers/multi_head_attention.py:74-76,171-173.  These are ~3 % of
// CoCa's FLOPs; the ViT and causal self-attention layers stay on the head_dim-64 kernels (attention.cu).
//
// Math: softmax(Q K^T * scale + mask) V with fp32 statistics, P rounded to bf16 for the PV product.  A fully masked
// query row yields zeros (SDPA would yield NaN; no caller on this path produces such a row).
#include "attention_generic.cuh"
#include "mmb200_internal.h"

namespace mmb {

namespace ag {

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

}  // namespace ag

// Row pitch D*2 + 16 bytes: an odd number of 16-byte chunks, so the 8 rows of an ldmatrix phase hit 8 distinct bank
// groups without a swizzle.
template <int D>
__global__ void __launch_bounds__(256) attn_fwd_generic_kernel(const AttnGenArgs p) {
  constexpr int PITCH = D * 2 + 16;
  constexpr int KS = D / 16;   // k-steps of Q K^T
  constexpr int NO = D / 8;    // 8-wide output column tiles
  extern __shared__ __align__(128) uint8_t gsm[];
  const int Sq_pad = (p.Sq + 15) & ~15, Skv_pad = (p.Skv + 63) & ~63;
  uint8_t* sQ = gsm;
  uint8_t* sK = sQ + Sq_pad * PITCH;
  uint8_t* sV = sK + Skv_pad * PITCH;
  const int b = blockIdx.x / p.H, h = blockIdx.x - b * p.H;
  const __nv_bfloat16* gq = p.q + b * p.bsq + h * D;
  const __nv_bfloat16* gk = p.k + b * p.bsk + h * D;
  const __nv_bfloat16* gv = p.v + b * p.bsv + h * D;
  constexpr int CH = D / 8;  // 16-byte chunks per row
  for (int i = threadIdx.x; i < Sq_pad * CH; i += blockDim.x) {
    const int r = i / CH, c = i - r * CH;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r < p.Sq) v = __ldg(reinterpret_cast<const uint4*>(gq + (long long)r * p.ldq + c * 8));
    *reinterpret_cast<uint4*>(sQ + r * PITCH + c * 16) = v;
  }
  for (int i = threadIdx.x; i < Skv_pad * CH; i += blockDim.x) {
    const int r = i / CH, c = i - r * CH;
    uint4 kk = make_uint4(0, 0, 0, 0), vv = kk;
    if (r < p.Skv) {
      kk = __ldg(reinterpret_cast<const uint4*>(gk + (long long)r * p.ldk + c * 8));
      vv = __ldg(reinterpret_cast<const uint4*>(gv + (long long)r * p.ldv + c * 8));
    }
    *reinterpret_cast<uint4*>(sK + r * PITCH + c * 16) = kk;
    *reinterpret_cast<uint4*>(sV + r * PITCH + c * 16) = vv;
  }
  __syncthreads();
  const uint32_t uQ = smem_u32(sQ), uK = smem_u32(sK), uV = smem_u32(sV);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const uint8_t* mrow_base = p.mask ? p.mask + b * p.mask_bs : nullptr;

  for (int qt = warp; qt < (Sq_pad >> 4); qt += nwarps) {
    const int q0 = qt * 16;
    uint32_t qa[KS][4];
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
      ag::ldsm_x4(qa[ks], uQ + (q0 + (lane & 7) + ((lane >> 3) & 1) * 8) * PITCH + (ks * 16 + (lane >> 4) * 8) * 2);
    float o[NO][4];
#pragma unroll
    for (int i = 0; i < NO; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    const int r0 = q0 + g, r1 = r0 + 8;
    // causal with Sq != Skv follows SDPA's is_causal (top-left aligned): key j visible to query i iff j <= i
    const int kv_end = p.causal ? min(p.Skv, q0 + 16) : p.Skv;
    const uint8_t* mr0 = mrow_base ? mrow_base + (long long)min(r0, p.Sq - 1) * p.mask_qs : nullptr;
    const uint8_t* mr1 = mrow_base ? mrow_base + (long long)min(r1, p.Sq - 1) * p.mask_qs : nullptr;

    for (int kvb = 0; kvb < kv_end; kvb += 64) {
      const int nt_valid = min(8, (kv_end - kvb + 7) >> 3);
      float s[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
        if (nt < nt_valid) {
#pragma unroll
          for (int kp = 0; kp < KS / 2; ++kp) {
            uint32_t kb[4];
            ag::ldsm_x4(kb, uK + (kvb + nt * 8 + (lane & 7)) * PITCH + (kp * 32 + (lane >> 3) * 8) * 2);
            ag::mma16816(s[nt], qa[2 * kp], kb[0], kb[1]);
            ag::mma16816(s[nt], qa[2 * kp + 1], kb[2], kb[3]);
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
          float v = s[nt][e] * p.scale_log2;
          bool ok = col < p.Skv && !(p.causal && col > row);
          if (ok && mrow_base) ok = ((e < 2) ? mr0 : mr1)[col] != 0;
          s[nt][e] = ok ? v : -INFINITY;
        }
        mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
        mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
      }
      mx0 = ag::quad_max(mx0);
      mx1 = ag::quad_max(mx1);
      const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
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
      for (int i = 0; i < NO; ++i) {
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
          for (int np = 0; np < NO / 2; ++np) {
            uint32_t vb[4];
            ag::ldsm_x4_t(vb, uV + (kvb + ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * PITCH + (np * 16 + (lane >> 4) * 8) * 2);
            ag::mma16816(o[2 * np], pa, vb[0], vb[1]);
            ag::mma16816(o[2 * np + 1], pa, vb[2], vb[3]);
          }
        }
      }
    }
    l0 = ag::quad_sum(l0);
    l1 = ag::quad_sum(l1);
    const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
    __nv_bfloat16* orow0 = p.out + b * p.bso + (long long)r0 * p.ldo + h * D;
    __nv_bfloat16* orow1 = p.out + b * p.bso + (long long)r1 * p.ldo + h * D;
#pragma unroll
    for (int nt = 0; nt < NO; ++nt) {
      if (r0 < p.Sq) *reinterpret_cast<uint32_t*>(orow0 + nt * 8 + 2 * t) = pack_bf16x2(o[nt][0] * i0, o[nt][1] * i0);
      if (r1 < p.Sq) *reinterpret_cast<uint32_t*>(orow1 + nt * 8 + 2 * t) = pack_bf16x2(o[nt][2] * i1, o[nt][3] * i1);
    }
  }
}

template <int D>
static int launch_generic(const AttnGenArgs& a, int B, cudaStream_t st) {
  const int Sq_pad = (a.Sq + 15) & ~15, Skv_pad = (a.Skv + 63) & ~63;
  const int smem = (Sq_pad + 2 * Skv_pad) * (D * 2 + 16);   // callers check generic_resident_fits()
  int warps = Sq_pad / 16;
  warps = warps < 1 ? 1 : (warps > 8 ? 8 : warps);
  cudaFuncSetAttribute(attn_fwd_generic_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  attn_fwd_generic_kernel<D><<<B * a.H, warps * 32, smem, st>>>(a);
  return (int)cudaGetLastError();
}



// ------------------------------------------------------------------------------------------------
// Attention PROBABILITIES on request: probs[b, h, i, j] = exp(q_i . k_j * scale - lse[b, h, i]) (0 where the key
// padding mask / causal mask removes the key), fp32 [B, H, S, S].  The fused attention kernels never materialise
// them; FLAVA's encoders return them (`TransformerOutput.attentions`, models/flava/transformer.py:255-293 via
// modules/layers/attention.py:220-239), so they are recomputed from the packed QKV and the row LSE the forward
// kernel already produced.  Memory-bound on the fp32 output (S*S*4 B per head); SIMT dot products from padded smem.
// Grid (ceil(S/32), H, B), 256 threads: 8 warps x 4 query rows, lanes over keys.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
attn_probs_kernel(const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ lse, const uint8_t* __restrict__ kmask,
                  float* __restrict__ probs, int S, int H, int causal, float scale_log2) {
  extern __shared__ uint8_t psm[];
  constexpr int PITCH = 144;                 // 64 bf16 + 16 B pad: 9 x 16 B per row -> conflict-free 16 B row reads
  uint8_t* sK = psm;                         // [S][PITCH]
  uint8_t* sQ = psm + (size_t)S * PITCH;     // [32][PITCH]
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int d = H * 64;
  const long long row0 = (long long)b * S;
  for (int idx = threadIdx.x; idx < S * 8; idx += 256) {          // K rows of this head: 8 x 16 B each
    const int j = idx >> 3, c = idx & 7;
    *reinterpret_cast<uint4*>(sK + j * PITCH + c * 16) =
        *reinterpret_cast<const uint4*>(qkv + (row0 + j) * 3 * d + d + h * 64 + c * 8);
  }
  for (int idx = threadIdx.x; idx < 32 * 8; idx += 256) {
    const int i = idx >> 3, c = idx & 7, qi = qb * 32 + i;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (qi < S) v = *reinterpret_cast<const uint4*>(qkv + (row0 + qi) * 3 * d + h * 64 + c * 8);
    *reinterpret_cast<uint4*>(sQ + i * PITCH + c * 16) = v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int rr = 0; rr < 4; ++rr) {
    const int i = warp * 4 + rr, qi = qb * 32 + i;
    if (qi >= S) break;
    float q[64];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const uint4 v = *reinterpret_cast<const uint4*>(sQ + i * PITCH + c * 16);   // broadcast
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) { q[c * 8 + 2 * e] = bf16_lo(w[e]); q[c * 8 + 2 * e + 1] = bf16_hi(w[e]); }
    }
    const float l2 = lse[((long long)b * H + h) * S + qi] * 1.4426950408889634f;
    float* out = probs + (((long long)b * H + h) * S + qi) * S;
    for (int j = lane; j < S; j += 32) {
      float acc = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint4 v = *reinterpret_cast<const uint4*>(sK + j * PITCH + c * 16);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          acc = fmaf(q[c * 8 + 2 * e], bf16_lo(w[e]), acc);
          acc = fmaf(q[c * 8 + 2 * e + 1], bf16_hi(w[e]), acc);
        }
      }
      const bool keep = (!causal || j <= qi) && (!kmask || kmask[row0 + j]);
      out[j] = keep ? ex2_approx(fmaf(acc, scale_log2, -l2)) : 0.f;
    }
  }
}

}  // namespace mmb

using namespace mmb;

extern "C" int mmb_attention_fwd_generic(const void* q, long long ldq, long long bsq, const void* k, long long ldk,
                                         long long bsk, const void* v, long long ldv, long long bsv, void* out,
                                         long long ldo, long long bso, const void* mask, long long mask_bs,
                                         long long mask_qs, int B, int Sq, int Skv, int H, int head_dim, int causal,
                                         float scale, void* stream) {
  if (B <= 0 || Sq <= 0 || Skv <= 0 || H <= 0) return MMB_ERR_ARG;
  if ((ldq | ldk | ldv | ldo | bsq | bsk | bsv | bso) & 7) return MMB_ERR_ARG;  // 16-byte vector loads / 4-byte stores
  AttnGenArgs a{};
  a.q = (const __nv_bfloat16*)q; a.k = (const __nv_bfloat16*)k; a.v = (const __nv_bfloat16*)v;
  a.out = (__nv_bfloat16*)out;
  a.ldq = ldq; a.ldk = ldk; a.ldv = ldv; a.ldo = ldo; a.bsq = bsq; a.bsk = bsk; a.bsv = bsv; a.bso = bso;
  a.mask = (const uint8_t*)mask; a.mask_bs = mask_bs; a.mask_qs = mask_qs;
  a.Sq = Sq; a.Skv = Skv; a.H = H; a.causal = causal;
  a.scale_log2 = scale * 1.4426950408889634f;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (head_dim != 64 && head_dim != 96 && head_dim != 128) return MMB_ERR_UNSUPPORTED;
  if (!generic_resident_fits(Sq, Skv, head_dim)) return attention_fwd_gstream(a, B, head_dim, st);
  switch (head_dim) {
    case 64: return launch_generic<64>(a, B, st);
    case 96: return launch_generic<96>(a, B, st);
    default: return launch_generic<128>(a, B, st);
  }
}

// 1 when the generic entry points run the streamed kernels (attention_generic_stream.cu) for this shape, else 0
extern "C" int mmb_attention_generic_streamed(int Sq, int Skv, int head_dim) {
  if (Sq <= 0 || Skv <= 0 || (head_dim != 64 && head_dim != 96 && head_dim != 128)) return 0;
  return generic_resident_fits(Sq, Skv, head_dim) ? 0 : 1;
}

// probs fp32 [B, H, S, S] from the packed QKV [B*S, 3*H*64] and the forward's row LSE [B, H, S] (head_dim 64).
extern "C" int mmb_attention_probs(const void* qkv, const float* lse, const unsigned char* kmask, float* probs, int B,
                                   int S, int H, int causal, float scale, void* stream) {
  if (B <= 0 || S <= 0 || H <= 0 || !qkv || !lse || !probs) return MMB_ERR_ARG;
  const int smem = (S + 32) * 144;
  if (smem > 200 * 1024) return MMB_ERR_UNSUPPORTED;
  cudaFuncSetAttribute(attn_probs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  attn_probs_kernel<<<dim3((S + 31) / 32, H, B), 256, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      (const __nv_bfloat16*)qkv, lse, kmask, probs, S, H, causal, scale * 1.4426950408889634f);
  return (int)cudaGetLastError();
}
