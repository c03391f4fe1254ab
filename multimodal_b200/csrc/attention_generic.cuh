// Arguments and dispatch of the general attention entry points (mmb_attention_fwd_generic / mmb_attention_bwd_generic):
// cross-attention, head_dim 64 / 96 / 128, batch-shared queries, boolean masks.  Two kernel families serve them:
//   attention_generic.cu / attention_generic_bwd.cu  the whole head's Q, K and V resident in shared memory (forward) and
//                                                     the SIMT backward, for the shapes generic_resident_fits() accepts;
//   attention_generic_stream.cu                       K / V (forward, dQ) and Q / dO (dK / dV) streamed through a
//                                                     shared-memory ring of constant size, for every longer shape.
#pragma once
#include "common.cuh"

namespace mmb {

struct AttnGenArgs {
  const __nv_bfloat16 *q, *k, *v;
  __nv_bfloat16* out;
  long long ldq, ldk, ldv, ldo;          // row strides (elements)
  long long bsq, bsk, bsv, bso;          // batch strides (elements); bsq = 0: queries shared by the whole batch
  const uint8_t* mask;                   // optional, 1 = attend
  long long mask_bs, mask_qs;            // mask[b*mask_bs + i*mask_qs + j]; mask_qs = 0: key mask [B, Skv]
  int Sq, Skv, H, causal;
  float scale_log2;
};

struct AttnGenBwdArgs {
  const __nv_bfloat16 *q, *k, *v, *dout;
  long long ldq, ldk, ldv, ldo;          // row strides (elements)
  long long bsq, bsk, bsv, bso;          // batch strides (elements); bsq = 0: queries shared by the whole batch
  const uint8_t* mask;                   // optional, 1 = attend: mask[b*mask_bs + i*mask_qs + j]
  long long mask_bs, mask_qs;
  __nv_bfloat16 *dq, *dk, *dv;           // bf16 outputs with the strides of q / k / v (dq may be NULL)
  float* dq_f32;                         // optional fp32 [Sq, ldq32] (+=): batch-shared queries, summed over the batch
  long long ldq32;
  float *lse, *dsum;                     // scratch [B, H, Sq]: row LSE (log2 units) and D_i
  int B, Sq, Skv, H, causal;
  float scale, scale_log2;
};

// The resident forward keeps Q (rows padded to 16) and K, V (rows padded to 64) of one head in shared memory, rows of
// 2*D + 16 bytes, within the 227 KB an H100 CTA can opt into.  Shapes that fit run the resident forward and the SIMT
// backward; all others run the streamed kernels in both directions.
inline bool generic_resident_fits(int Sq, int Skv, int D) {
  const long long rows = ((Sq + 15LL) & ~15LL) + 2 * ((Skv + 63LL) & ~63LL);
  return rows * (2LL * D + 16) <= 227LL * 1024;
}

// attention_generic_stream.cu; D in {64, 96, 128}, B and H at most 65535 (MMB_ERR_UNSUPPORTED beyond)
int attention_fwd_gstream(const AttnGenArgs& a, int B, int D, cudaStream_t stream);
int attention_bwd_gstream(const AttnGenBwdArgs& a, int D, cudaStream_t stream);

}  // namespace mmb
