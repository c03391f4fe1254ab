// Internal constants shared by the kernels of libmmb200.so (the public C ABI is include/mmb200.h).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define MMB_OK 0
#define MMB_ERR_ARG (-22)          /* -EINVAL: bad pointer alignment / leading dimension / shape */
#define MMB_ERR_UNSUPPORTED (-95)  /* -EOPNOTSUPP: shape or mode not implemented (never falls back) */
#define MMB_ERR_DRIVER (-5)        /* -EIO: CUDA driver entry point / tensor-map encode failed */

// GEMM epilogues
#define EPI_BF16 0       /* D0 = bf16(alpha*acc + bias) */
#define EPI_BF16_ACT 1   /* D0 = bf16(pre), D1 = bf16(act(D0)), pre = alpha*acc + bias */
#define EPI_BF16_DACT 2  /* D0 = bf16(alpha*acc * act'(aux)) */
#define EPI_F32 3        /* D0 = fp32(alpha*acc + bias), optional reduce-add (split-K / accumulate) */
#define EPI_CE_STATS 4   /* no tensor output: per (row, 128-column part) online-softmax statistics of T*acc */
#define EPI_CE_GRAD 5    /* D0 = bf16(d loss / d acc) of the temperature-scaled cross-entropy, from T*acc in registers */

#define ACT_QUICK_GELU 0
#define ACT_GELU_ERF 1
#define ACT_RELU 2

namespace mmb {
int make_tmap_2d(CUtensorMap* out, const void* ptr, int elem_bytes, bool is_f32, uint64_t inner, uint64_t outer,
                 uint64_t pitch_bytes, uint32_t box_inner, uint32_t box_outer);
int make_tmap_3d_bf16(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t dim1, uint64_t dim2, uint64_t pitch1,
                      uint64_t pitch2, uint32_t box_inner, uint32_t box1);
int num_sms();
}  // namespace mmb

// Deterministic reductions: no floating-point atomics anywhere, so a run's results do not depend on the order in which
// CTAs happen to finish.  Kernels write per-CTA (or per-row-slice) partials into scratch and a fixed-order reduction
// adds them into the output.
namespace mmb {
// Device scratch of at least `bytes`, private to (device, stream, slot); grows on demand (cudaFree synchronises, so a
// buffer an earlier launch still uses is never freed under it).  nullptr if the allocation fails.
void* scratch(int slot, size_t bytes, cudaStream_t stream);
// SCR_ATTN_D: rowsum(dO * O) of the streamed attention backward, fp32 [B*H*S], written by its dQ kernel and read by its
// dK / dV kernel.  SCR_ATTN_DQ: fp32 per-batch-chunk sums of dQ of the streamed general attention backward
// (attention_generic_stream.cu), added into dq_f32 in chunk order.  SCR_ATTN_DEC: fp32 per-split partials (O, m, l) of
// the split-KV decode attention (attention_decode.cu), added in split order by its combine kernel.  SCR_PATCH_DROP: the
// keep-index inverse map and the position / mask-token partials of the gathered token-assembly backward (patch_drop.cu)
enum ScratchSlot { SCR_GEMM_SPLITK = 0, SCR_GEMM_COLSUM, SCR_LN_BWD, SCR_COLSUM, SCR_BATCH_SUM, SCR_LOSS, SCR_ATTN_D,
                   SCR_ATTN_DQ, SCR_ATTN_DEC, SCR_PATCH_DROP, SCR_COUNT };
// out[n] (+)= sum_{p = 0..P-1} part[p * ldp + n] for n < N, summed in increasing p (accumulate = 0: out is overwritten).
int reduce_partials(const float* part, int P, int N, long long ldp, float* out, int accumulate, cudaStream_t stream);
}  // namespace mmb
