/* libmmb200 — C ABI of the H100-native (sm_90a) dual-encoder + contrastive-loss hot path.
 *
 * The reference (facebookresearch/multimodal) has no FFI: its hot path is Python calling
 * torch.nn.functional.  These entry points are what a maintainer would bind (ctypes; see
 * INTEGRATION.md) to replace each library call on that path.  Conventions:
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless noted;
 *   - `stream` is a cudaStream_t passed as void*; every call is asynchronous on that stream;
 *   - row-major tensors with explicit leading dimensions (in ELEMENTS);
 *   - return value: 0 on success, a positive cudaError_t, or a negative MMB_ERR_* code.
 *     There is no CPU fallback: unsupported shapes return MMB_ERR_UNSUPPORTED.
 */
#ifndef MMB200_H_
#define MMB200_H_
#ifdef __cplusplus
extern "C" {
#endif

#define MMB_OK 0
#define MMB_ERR_ARG (-22)
#define MMB_ERR_UNSUPPORTED (-95)
#define MMB_ERR_DRIVER (-5)

/* GEMM epilogues (mmb_gemm_bf16) */
#define MMB_EPI_BF16 0      /* D0 = bf16(alpha*acc + bias)                                   */
#define MMB_EPI_BF16_ACT 1  /* D0 = bf16(pre = alpha*acc + bias), D1 = bf16(act(D0))         */
#define MMB_EPI_BF16_DACT 2 /* D0 = bf16(alpha*acc * act'(aux)); ReLU: aux > 0 ? alpha*acc : +0 */
#define MMB_EPI_F32 3       /* D0 = fp32(alpha*acc + bias) (+ D0 when accumulate); split-K summed in a fixed order */
#define MMB_ACT_QUICK_GELU 0 /* torchmultimodal/modules/layers/activation.py:12-25 ("SiLU")  */
#define MMB_ACT_GELU_ERF 1   /* nn.GELU(), torchmultimodal/modules/layers/mlp.py             */
#define MMB_ACT_RELU 2       /* nn.ReLU(), the default of MLP and the transformer layers      */

int mmb_version(void);

/* D[M,N] = alpha * A (x) B (+ bias[N]), bf16 operands, fp32 accumulation on Hopper tensor cores (wgmma).
 *   a_mn_major = 0: A is [M,K] row-major (lda >= K);  1: A is stored [K,M] row-major (lda >= M)
 *   b_mn_major = 0: B is [N,K] row-major (ldb >= K);  1: B is stored [K,N] row-major (ldb >= N)
 * Replaces: F.linear in torch/nn/functional.py:6478 (in-proj), :6690 (out-proj),
 *           torch/nn/modules/transformer.py:980-982 (linear1/linear2), their autograd dgrad/wgrad,
 *           torch.matmul in modules/losses/contrastive_loss_with_temperature.py:90-95,
 *           `x @ self.projection` in models/clip/image_encoder.py:112, Linear in text_encoder.py:130.
 * colsum (optional, EPI_BF16 / EPI_BF16_DACT): colsum[n] += sum_m of the bf16-rounded D0[m,n] — the bias gradient of
 *           the Linear whose input-gradient this GEMM produces (linear1.bias from the FC2 dgrad), fused into the
 *           epilogue's copy-out so the tensor is not re-read by a column-sum pass.
 * accumulate is accepted with EPI_F32 only, bias with every epilogue but EPI_BF16_DACT; either elsewhere: MMB_ERR_ARG. */
int mmb_gemm_bf16(const void* A, long long lda, int a_mn_major, const void* B, long long ldb, int b_mn_major,
                  void* D0, long long ldd0, void* D1, long long ldd1, int M, int N, int K, int epilogue, int act,
                  float alpha, const float* bias, const void* aux, long long ld_aux, int splits, int accumulate,
                  float* colsum, void* stream);

/* Test / A-B hook (process-wide): force the kernel variant mmb_gemm_bf16 dispatches to.
 *   cta2: -1 = automatic (size heuristic), 0 = one CTA per 128x256 tile, 1 = 2-CTA clusters (256x256 tiles, the B tile
 *   multicast to both CTAs); epilogue_warps: 0 or 8 (the two consumer warpgroups run every epilogue).  Returns
 *   MMB_ERR_ARG on other values.
 * No reference counterpart: it exists so the parity tests can drive both kernels over every operand / epilogue case. */
int mmb_gemm_set_mode(int cta2, int epilogue_warps);

/* ---- fused similarity GEMM + temperature-scaled cross-entropy: the logits never reach HBM ---------------------------
 * Replaces `torch.matmul(a, b_all.T) * exp(logit_scale)` + `F.cross_entropy` of
 * modules/losses/contrastive_loss_with_temperature.py:90-107 (and serves any Linear -> CrossEntropy head).
 * A [M,K], B [N,K] bf16 row-major; logits[m,n] = exp(*log_scale) * sum_k A[m,k] B[n,k] live in registers only.
 *
 * mmb_gemm_ce_stats: online-softmax statistics.  For every row m and every 128-column part of this launch it writes one
 *   float4 {max, sum e^(x-max), sum e^(x-max) x, sum x} into part[m * part_ld + part0 + ...] (mmb_gemm_ce_num_parts(N)
 *   entries per row and launch), and xlabel[m] = logits[m, label0 + m] when that column exists in this launch.  Several
 *   launches (one per peer GPU's column block, B read in place from the peer's buffer) fill disjoint part ranges.
 * mmb_ce_stats_reduce: combines a row's parts into lse_out[m], row_loss[m] (label smoothing, optional masked-mean row
 *   weights) and accumulates loss_weight * d(mean loss)/d(log_scale) into dscale_accum.
 * mmb_gemm_ce_grad: recomputes the logits tile and writes d(loss_weight * mean CE)/d(sims) in bf16 (the operand of the
 *   embedding-gradient GEMMs); columns [col_lo, col_hi) additionally receive the other direction's transposed term
 *   rebuilt from lse_col (GLOBAL / LOCAL backprop without a reduce-scatter, see DESIGN.md §4). */
int mmb_gemm_ce_num_parts(int N);
int mmb_gemm_ce_stats(const void* A, long long lda, const void* B, long long ldb, int M, int N, int K,
                      const float* log_scale, int label0, void* part, int part_ld, int part0, float* xlabel, void* stream);
int mmb_ce_stats_reduce(const void* part, int part_ld, int n_parts, const float* xlabel, int rows, int n_total,
                        float label_smoothing, float loss_weight, const float* row_w, float* row_loss, float* lse_out,
                        float* dscale_accum, void* stream);
/* Vocabulary heads (Linear -> nn.CrossEntropyLoss(ignore_index), models/coca/coca_model.py:443-454): the same fused
 * statistics GEMM with an explicit int32 label column per row, and the reduce that yields accum[0] += sum of the kept
 * rows' losses, accum[1] += their count (mean = accum[0] / accum[1]); rows whose label == ignore_index are skipped. */
int mmb_gemm_ce_stats_labels(const void* A, long long lda, const void* B, long long ldb, int M, int N, int K,
                             const float* log_scale, const int* labels, void* part, int part_ld, int part0,
                             float* xlabel, void* stream);
int mmb_ce_labels_reduce(const void* part, int part_ld, int n_parts, const float* xlabel, const int* labels,
                         int ignore_index, int rows, float* row_loss, float* accum, void* stream);
int mmb_gemm_ce_grad(const void* A, long long lda, const void* B, long long ldb, int M, int N, int K,
                     const float* log_scale, int label0, int n_total, int rows_total, float label_smoothing,
                     float loss_weight, const float* lse_row, const float* row_w, const float* lse_col,
                     const float* col_w, int col_lo, int col_hi, void* dsims_bf16, long long ldd, void* stream);


/* ---- HBM-bound kernels ------------------------------------------------------------------------------------ */

/* dst[i] = bf16(src[i]) — parameter shadow for the tensor-core operands (what torch.autocast does per call). */
int mmb_cast_f32_to_bf16(const float* src, void* dst_bf16, long long n, void* stream);
/* bf16 -> fp32 (result of the optional bf16-compressed gradient all-reduce back into the optimizer's fp32 input). */
int mmb_cast_bf16_to_f32(const void* src, float* dst, long long n, void* stream);
/* mmb_cast_f32_to_bf16 with a per-sample stochastic-depth factor: dst[i] = bf16(fl32(scale[i / per_scale] * src[i]));
 * per_scale (elements per factor, e.g. S*d) > 0 and a multiple of 4.  The gradient entering the last layer's MLP branch
 * of a stack without a final LayerNorm (StochasticDepth(p, "row"), modules/layers/transformer.py:63-70). */
int mmb_cast_f32_to_bf16_scaled(const float* src, void* dst_bf16, long long n, const float* scale, long long per_scale,
                                void* stream);

/* Patch im2col + cast: img fp32 [B,3,H,W] -> bf16 [B*(H/ps)*(W/ps), 3*ps*ps] with row pitch ld_out elements (>= 3*ps*ps;
 * a multiple of 8 keeps the rows TMA-addressable, e.g. 592 for 14x14 patches), K order (c,kh,kw), patches row-major.
 * Replaces the data movement half of nn.Conv2d(3,width,ps,ps,bias=False), models/clip/image_encoder.py:50-56,91-97. */
int mmb_im2col_patches(const float* img, void* out_bf16, long long ld_out, int B, int H, int W, int ps, void* stream);

/* x_out = x_in (+ y_bf16); ln = LayerNorm(x_out)*gamma+beta, fp32 statistics.  Any of x_in/y/x_out/ln_bf16/ln_f32/
 * mean/rstd may be NULL.  rows_per_group > 0 selects the gather mode: logical row m reads physical row
 * m*rows_per_group + (row_idx ? row_idx[m] : 0) and every output is written compactly at row m.
 * Replaces: residual add + norm1/norm2 (torch/nn/modules/transformer.py:946-951), Fp32LayerNorm ln_post / ln_final
 * (torchmultimodal/modules/layers/normalizations.py:17-25; models/clip/image_encoder.py:111, text_encoder.py:125). */
int mmb_add_layernorm_fwd(const float* x_in, const void* y_bf16, float* x_out, void* ln_bf16, float* ln_f32,
                          const float* gamma, const float* beta, float* mean, float* rstd, const int* row_idx,
                          int rows_per_group, int M, int d, float eps, void* stream);
/* mmb_add_layernorm_fwd with stochastic depth on the added branch (torchvision stochastic_depth(y, p, "row") as
 * TransformerEncoderLayer(drop_path_rate=...) applies it, modules/layers/transformer.py:63-70,95-129):
 * x_out = x_in + fl32(scale[m / rows_per_scale] * y) for row m; scale fp32 [M / rows_per_scale] holds the drawn noise
 * (0 or 1/(1-p)); the LayerNorm is unchanged.  y and scale required, rows_per_scale > 0, no row gather. */
int mmb_add_layernorm_fwd_scaled(const float* x_in, const void* y_bf16, float* x_out, void* ln_bf16, float* ln_f32,
                                 const float* gamma, const float* beta, float* mean, float* rstd, const float* scale,
                                 int rows_per_scale, int M, int d, float eps, void* stream);

/* CLIP ViT token assembly + ln_pre: x0 = LN(cat(cls, patch_out) + pos) (models/clip/image_encoder.py:94-106). */
int mmb_vit_embed_ln_fwd(const void* patch_out_bf16, const float* cls, const float* pos, const float* gamma,
                         const float* beta, float* x0, float* mean, float* rstd, int B, int S, int d, float eps,
                         void* stream);

/* LayerNorm backward (+ residual-gradient add): g_out = (g_in?) + dLN/dx; dgamma/dbeta accumulated (+=) in a fixed order.
 * dy is bf16 or fp32 (exactly one non-NULL).  Gather mode as in the forward: x/dy/mean/rstd are compact [M,d],
 * g_out/g_bf16 are scattered to the physical rows of a zero-initialised [*,d] buffer.
 * gsum (optional, needs g_bf16): gsum[c] += sum over rows of the bf16-rounded g — the bias gradient of the Linear layer
 * whose backward consumes g_bf16 next (out_proj / linear2 in torch/nn/modules/transformer.py:961-982), fused here so
 * that tensor is not re-read by a column-sum kernel. */
int mmb_layernorm_bwd(const float* x, const void* dy_bf16, const float* dy_f32, const float* mean, const float* rstd,
                      const float* gamma, const float* g_in, float* g_out, void* g_bf16, float* dgamma, float* dbeta,
                      const int* row_idx, int rows_per_group, int M, int d, float* gsum, void* stream);
/* mmb_layernorm_bwd for a residual stream whose next branch was scaled by stochastic depth: g_out is unchanged,
 * g_bf16 = bf16(fl32(scale[m / rows_per_scale] * g_out)) (the gradient that enters the branch) and gsum sums those
 * scaled bf16 values.  g_bf16 and scale required, rows_per_scale > 0, no row scatter. */
int mmb_layernorm_bwd_scaled(const float* x, const void* dy_bf16, const float* dy_f32, const float* mean,
                             const float* rstd, const float* gamma, const float* g_in, float* g_out, void* g_bf16,
                             float* dgamma, float* dbeta, const float* scale, int rows_per_scale, int M, int d,
                             float* gsum, void* stream);

/* Backward of mmb_vit_embed_ln_fwd: dt = d/d(cat+pos) fp32 [B,S,d]; dpatch = bf16 copy of rows s>=1, compact. */
int mmb_vit_embed_ln_bwd(const void* patch_out_bf16, const float* cls, const float* pos, const float* dy_f32,
                         const float* mean, const float* rstd, const float* gamma, float* dt_f32, void* dpatch_bf16,
                         float* dgamma, float* dbeta, int B, int S, int d, void* stream);

/* out[j] += sum_b in[b*ld + j], j < n   (positional-embedding / cls gradients) */
int mmb_batch_sum(const float* in, float* out, int Bn, long long ld, int n, void* stream);
/* out[n] += sum_m x[m*ld + n]           (bias gradients), x bf16 */
int mmb_colsum_bf16(const void* x_bf16, float* out, int M, int N, long long ld, void* stream);

/* x[b,s,:] = emb[tokens[b,s],:] + pos[s,:]; tokens int64, bit-exact gather (models/clip/text_encoder.py:118-119). */
int mmb_text_embed_fwd(const long long* tokens, const float* emb, const float* pos, float* x, int B, int S, int d,
                       int V, void* stream);
int mmb_text_embed_bwd(const long long* tokens, const float* g, float* demb, int B, int S, int d, void* stream);
/* idx[b] = argmax_s tokens[b,s], first maximum (EOT position; models/clip/text_encoder.py:130-132). Bit-exact. */
int mmb_argmax_tokens(const long long* tokens, int* idx, int B, int S, void* stream);

/* F.normalize(x, dim=1, eps) (models/clip/model.py:72-73) and its backward. */
int mmb_l2norm_fwd(const float* x, float* y, void* y_bf16, float* inv_norm, int B, int E, float eps, void* stream);
int mmb_l2norm_bwd(const float* dy, const float* y, const float* inv_norm, float* dx, void* dx_bf16, int B, int E,
                   void* stream);

/* Fused AdamW over a flat buffer (torch.optim.AdamW update rule); writes the bf16 shadow and optionally zeroes g. */
int mmb_adamw_step(float* p, float* g, float* m, float* v, void* p_bf16, long long n, float lr, float beta1,
                   float beta2, float eps, float weight_decay, int step, float grad_scale, int zero_grad,
                   void* stream);

/* AnyPrecisionAdamW.step for ONE fp32 parameter tensor (modules/optimizers/anyprecision.py:99-199): momentum /
 * variance / Kahan-compensation buffers in caller-chosen dtypes (*_dtype: 0 = fp32, 1 = bf16; reference defaults: fp32
 * momentum, bf16 variance, bf16 compensation).  comp == NULL selects the plain update (use_kahan_summation=False).
 * Every in-place rounding of the reference is reproduced; one fused pass replaces its ~12 elementwise kernels.
 * p_bf16 (optional): bf16 copy of the updated weights (the GEMM operand shadow); zero_grad clears g in the same pass;
 * grad_scale multiplies g first (1/world after a summed all-reduce; the reference has no such factor: pass 1). */
int mmb_anyprecision_adamw_step(float* p, float* g, void* m, int m_dtype, void* v, int v_dtype, void* comp,
                                int comp_dtype, void* p_bf16, long long n, double lr, double beta1, double beta2,
                                double eps, double weight_decay, int step, float grad_scale, int zero_grad,
                                void* stream);
int mmb_memset_async(void* p, int value, long long bytes, void* stream);
/* Standalone activation, fp32: kind MMB_ACT_QUICK_GELU = x*sigmoid(1.702x) (modules/layers/activation.py:24-25),
 * MMB_ACT_GELU_ERF = nn.GELU(), MMB_ACT_RELU = max(x, 0) (exact).  (Inside the encoders the activation is a GEMM
 * epilogue.) */
int mmb_act_fwd(const float* x, float* y, long long n, int kind, void* stream);

/* ---- attention --------------------------------------------------------------------------------------------- */
/* O = softmax(Q K^T * scale [+ causal mask]) V per (batch, head), head_dim 64, any S (tensor-core kernels: one CTA per
 * head with the whole head in shared memory up to S = 384, K / V streamed through shared memory above); qkv bf16
 * [B*S, 3*H*64] packed [q|k|v], out bf16 [B*S, H*64], lse fp32 [B,H,S] in natural-log units (may be NULL for
 * forward-only callers; a row with no visible key gets O = 0 and lse = -inf).  B and H are at most 65535 above S = 384.
 * Replaces F.scaled_dot_product_attention (torch/nn/functional.py:6682). */
int mmb_attention_fwd(const void* qkv, void* out, float* lse, int B, int S, int H, int head_dim, int causal,
                      float scale, void* stream);
int mmb_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv, int B, int S,
                      int H, int head_dim, int causal, float scale, void* stream);
/* Number of kernels one mmb_attention_bwd(_kmask) call launches at sequence length S — for callers that count launches.
 * 1 up to S = 384 (one kernel computes dQ, dK and dV); 2 above (a dQ kernel that also writes rowsum(dO * O) to library
 * scratch, then a dK / dV kernel), both deterministic without atomics. */
int mmb_attention_bwd_launches(int S);

/* Same with a key-padding mask [B,S] (1 = attend, 0 = masked_fill(-inf)): the BERT-style attention of the FLAVA text
 * tower (modules/encoders/bert_text_encoder.py:87-93 -> modules/layers/attention.py:228-229).  Any S, as above. */
int mmb_attention_fwd_kmask(const void* qkv, void* out, float* lse, const unsigned char* kmask, int B, int S, int H,
                            int head_dim, int causal, float scale, void* stream);

/* Attention probabilities on request: probs fp32 [B,H,S,S] = exp(q.k*scale - lse) (0 where masked), recomputed from the
 * packed QKV and the row LSE written by mmb_attention_fwd*.  Serves `TransformerOutput.attentions` of the FLAVA
 * encoders (models/flava/transformer.py:255-293; modules/layers/attention.py:220-239 returns the softmax output). */
int mmb_attention_probs(const void* qkv, const float* lse, const unsigned char* kmask, float* probs, int B, int S, int H,
                        int causal, float scale, void* stream);

/* ---- FLAVA encoder front/back ends (config 3, forward) -------------------------------------------------------- */
/* x = LayerNorm(word[ids] + pos[arange(S)] + type[type_ids or 0]) — BERTTextEmbeddings.forward,
 * modules/layers/text_embedding.py:70-104.  ids/type_ids int64 (bit-exact gathers).  kmask_out (optional) receives
 * ids != pad_id, the default padding mask of BERTTextEncoder.forward (bert_text_encoder.py:87-90). */
int mmb_bert_embed_ln_fwd(const long long* ids, const long long* type_ids, const float* word, const float* pos,
                          const float* type, const float* gamma, const float* beta, float* x, unsigned char* kmask_out,
                          long long pad_id, int B, int S, int d, int V, float eps, void* stream);
/* x = cat(cls, mask ? mask_token : patch_out) + pos — ImageEmbeddings.forward, models/flava/image_encoder.py:139-175,
 * and PatchEmbeddings.forward, modules/layers/patch_embedding.py:104-154 (cls = NULL: include_cls_embed=False, S = P). */
int mmb_vit_assemble_fwd(const void* patch_out_bf16, const float* cls, const float* pos, const float* mask_token,
                         const unsigned char* patch_mask, float* x, int B, int S, int d, void* stream);
/* out[b,:] = bf16(x[b*rows_per_group + row, :]) — `hidden[:, 0]` selects (Pooler, projections; losses/flava.py:92-96). */
int mmb_gather_rows_cast(const float* x, void* out_bf16, int B, int rows_per_group, int row, int d, void* stream);
/* out[m,:] = bf16(x[idx[m]*ld : +d]), idx int64 flat row numbers: the boolean-mask select `hidden_states[masked_tokens, :]`
 * of MaskedPredictionLoss.forward (modules/losses/flava.py:212-215) and `multimodal_masked_sequence[pos_mask]` (:430). */
int mmb_gather_rows_idx_cast(const float* x, long long ld, const long long* idx, void* out_bf16, int n, int d, void* stream);
int mmb_tanh_inplace(float* x, long long n, void* stream);
/* out[b] = cat([cls], a[b], b[b]) along tokens — models/flava/transformer.py:55-58 + model.py:294-297. */
int mmb_concat_tokens(const float* cls, const float* a, const float* b, float* out, int B, int Sa, int Sb, int d,
                      void* stream);


/* ---- FLAVA encoders, backward (config 3 as a training step; autograd of the files cited on the forward entries) -- */
/* Backward of mmb_attention_fwd_kmask (any S): masked keys get P = dS = 0, i.e. zero dK / dV rows. */
int mmb_attention_bwd_kmask(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                            const unsigned char* kmask, int B, int S, int H, int head_dim, int causal, float scale,
                            void* stream);
/* Backward of mmb_bert_embed_ln_fwd: the pre-LayerNorm sum and its statistics are recomputed from the tables; dx is
 * scatter-added into dword[ids] / dpos[s] / dtype[type_ids], dgamma / dbeta are accumulated (all fp32, += ). */
int mmb_bert_embed_ln_bwd(const long long* ids, const long long* type_ids, const float* word, const float* pos,
                          const float* type, const float* gamma, const float* dy, float* dword, float* dpos, float* dtype,
                          float* dgamma, float* dbeta, int B, int S, int d, int V, float eps, void* stream);
/* Backward of mmb_vit_assemble_fwd for the patch rows: dpatch[b*P+p] = bf16(mask ? 0 : g[b,off+p]) (the operand of the
 * patch-projection weight gradient), dmask_token += sum of the masked rows' g.  dcls / dpos: mmb_batch_sum of g. */
int mmb_vit_assemble_bwd(const float* g, const unsigned char* patch_mask, void* dpatch_bf16, float* dmask_token, int B,
                         int S, int d, int has_cls, void* stream);
/* ---- Random patch dropping (FLIP: PatchEmbeddings(patch_drop_rate=...), modules/layers/patch_embedding.py:104-154,
 * modules/masking/random_masking.py).  keep: int32 [B, L], per sample L distinct patch indices in [0, P) in the order
 * the tokens take (an index outside [0, P) traps).  P = (H/ps)*(W/ps); off = 1 with a CLS token, else 0. */
/* mmb_im2col_patches on the kept patches only: out row b*L+j = patch keep[b,j] of image b (same K order and pitch). */
int mmb_im2col_patches_gather(const float* img, const int* keep, void* out_bf16, long long ld_out, int B, int H, int W,
                              int ps, int L, void* stream);
/* x [B, off+L, d] fp32: x[b,0] = cls + pos[0] (cls != NULL); x[b,off+j] = (mask[b,p] ? mask_token : patch_out[b*L+j])
 * + pos[off+p], p = keep[b,j]; patch_out bf16 [B*L, d], patch_mask uint8 [B, P] (optional, indexed by patch). */
int mmb_vit_assemble_gather_fwd(const void* patch_out_bf16, const float* cls, const float* pos, const float* mask_token,
                                const unsigned char* patch_mask, const int* keep, float* x, int B, int L, int P, int d,
                                void* stream);
/* Backward of mmb_vit_assemble_gather_fwd from g fp32 [B, off+L, d]: dpatch[b*L+j] = bf16(mask ? 0 : g[b,off+j]);
 * dmask_token += sum of the masked kept rows; dcls += sum_b g[b,0]; dpos[0] += sum_b g[b,0] (with cls) and
 * dpos[off+p] += sum over the samples b that kept p of g[b, off+j(b,p)] (+= 0 for a patch no sample kept).  dmask_token,
 * dcls and dpos may each be NULL.  No atomics: the sums run in a fixed order, run-to-run bit-identical. */
int mmb_vit_assemble_gather_bwd(const float* g, const unsigned char* patch_mask, const int* keep, void* dpatch_bf16,
                                float* dmask_token, float* dcls, float* dpos, int B, int L, int P, int d, int has_cls,
                                void* stream);
/* Inverse of mmb_concat_tokens for gradients: g [B, cls+Sa+Sb, d] fp32 -> bf16 [B*Sa, d] and [B*Sb, d]. */
int mmb_split_tokens_cast(const float* g, void* a_bf16, void* b_bf16, int B, int Sa, int Sb, int d, int has_cls,
                          void* stream);
/* dx = dy * (1 - y^2), y = tanh(x) (Pooler, modules/losses/flava.py:92-96); fp32 and / or bf16 output. */
int mmb_tanh_bwd(const float* dy, const float* y, float* dx, void* dx_bf16, long long n, void* stream);
/* dst[b*rows_per_group + row, :] += src[b, :] — gradient of the `hidden[:, row]` select (mmb_gather_rows_cast). */
int mmb_scatter_rows_add(const float* src, float* dst, int B, int rows_per_group, int row, int d, void* stream);
/* dst[idx[m]*ld : +d] += src[m, :] (atomics; idx may repeat) — gradient of mmb_gather_rows_idx_cast. */
int mmb_scatter_rows_idx_add(const float* src, const long long* idx, float* dst, long long ld, int n, int d, void* stream);
/* d loss / d logits (bf16) of the label-indexed mean cross-entropy of mmb_ce_labels: w * (softmax - onehot) for kept rows,
 * 0 for ignored rows, w = grad_scale * (grad_scale_dev ? *grad_scale_dev : 1) / max(accum[1], 1) (accum = the forward's
 * {sum, count}; NULL: count 1; grad_scale_dev: the incoming d loss as a device scalar, no host sync). */
int mmb_ce_labels_bwd(const float* logits, long long ld, const long long* labels, long long label_stride,
                      long long ignore_index, int M, int V, const float* accum, float grad_scale,
                      const float* grad_scale_dev, void* dlogits_bf16, long long ldd, void* stream);
/* dx = bf16(dy * act'(pre)), bf16 tensors of n elements; kind = ACT_QUICK_GELU (0) / ACT_GELU_ERF (1) / ACT_RELU (2,
 * dx = pre > 0 ? dy : +0 exactly): the activation
 * backward outside a GEMM epilogue (MaskedPredictionHead transform, modules/losses/flava.py:174-180 under autograd). */
int mmb_act_bwd(const void* dy_bf16, const void* pre_bf16, void* dx_bf16, long long n, int kind, void* stream);

/* ---- CoCa forward helpers (SURVEY.md §8 a14) ------------------------------------------------------------------ */
/* x[b,s] = emb[ids[b,s]] + pos[s] (s < S-1), x[b,S-1] = cls + pos[S-1]; ids is [B, S-1] when cls != NULL, else [B, S]
 * — CoCaTextEmbeddings.forward, models/coca/text_decoder.py:48-60. */
int mmb_coca_text_embed_fwd(const long long* ids, const float* emb, const float* cls, const float* pos, float* x, int B,
                            int S, int d, int V, void* stream);
/* softmax(Q K^T * scale + mask) V for cross-attention / head_dim 64, 96, 128 / batch-shared queries / boolean masks:
 * F.scaled_dot_product_attention at modules/layers/multi_head_attention.py:74-76,171-173.  q,k,v,out are bf16 with row
 * strides ld* and batch strides bs* (elements, multiples of 8; bsq = 0 shares the queries across the batch); head h
 * occupies columns [h*head_dim, (h+1)*head_dim).  mask (optional, uint8, 1 = attend) is addressed
 * mask[b*mask_bs + i*mask_qs + j] (mask_qs = 0: key-padding mask).  causal follows SDPA's is_causal (j <= i).
 * Any Sq and Skv.  Shapes whose Q, K and V of one head fit in a CTA's shared memory,
 * (pad16(Sq) + 2*pad64(Skv)) * (2*head_dim + 16) <= 227 KB, run a kernel that keeps the head resident; longer ones run
 * tensor-core kernels that stream K / V through shared memory (mmb_attention_generic_streamed tells which).  A query
 * row with no visible key gets O = 0.  On the streamed path B and H are at most 65535 (MMB_ERR_UNSUPPORTED beyond) and
 * q, k, v and out must be 16-byte aligned (MMB_ERR_ARG otherwise). */
int mmb_attention_fwd_generic(const void* q, long long ldq, long long bsq, const void* k, long long ldk, long long bsk,
                              const void* v, long long ldv, long long bsv, void* out, long long ldo, long long bso,
                              const void* mask, long long mask_bs, long long mask_qs, int B, int Sq, int Skv, int H,
                              int head_dim, int causal, float scale, void* stream);
/* Backward of mmb_attention_fwd_generic (same addressing, any Sq and Skv).  The shapes the resident forward serves run
 * SIMT kernels in fp32 arithmetic; longer ones run the streamed tensor-core kernels (two launches, a third for dq_f32),
 * so a forward and its backward always take the same path.  dq / dk / dv (bf16) use the strides of q / k / v; dq_bf16
 * may be NULL; on the streamed path dq / dk / dv must be 16-byte aligned (MMB_ERR_ARG otherwise).  dq_f32 (optional, fp32 [Sq, ldq32], += : zero it first) receives the gradient of batch-shared queries
 * (bsq = 0) summed over the batch: with fp32 atomics on the resident path, and run-to-run deterministic on the streamed
 * path (per-batch-chunk sums in library scratch, chunks sized from the shape alone, added in a fixed order).  A masked
 * key gets zero dK / dV rows and a query row with no visible key a zero dQ row.  scratch: fp32 [2 * B * H * Sq] (row
 * LSE and rowsum(P * dP)).  Autograd of F.scaled_dot_product_attention at
 * modules/layers/multi_head_attention.py:74-76,171-173 for the CoCa poolers / decoders and the standalone layers. */
int mmb_attention_bwd_generic(const void* q, long long ldq, long long bsq, const void* k, long long ldk, long long bsk,
                              const void* v, long long ldv, long long bsv, const void* dout, long long ldo, long long bso,
                              const void* mask, long long mask_bs, long long mask_qs, void* dq_bf16, float* dq_f32,
                              long long ldq32, void* dk_bf16, void* dv_bf16, float* scratch, int B, int Sq, int Skv, int H,
                              int head_dim, int causal, float scale, void* stream);
/* 1 when mmb_attention_fwd_generic / mmb_attention_bwd_generic run the streamed kernels for this shape (the head does not
 * fit in shared memory), 0 when they run the resident forward and SIMT backward or head_dim is unsupported.  Host only. */
int mmb_attention_generic_streamed(int Sq, int Skv, int head_dim);
/* Decode attention: mmb_attention_fwd_generic's arguments and result for Sq <= 16 query rows over any number of keys
 * (the autoregressive step of MultiHeadAttentionWithCache with a key / value cache,
 * modules/layers/multi_head_attention.py:152-175).  The keys are split across CTAs (grid splits x H x B,
 * mmb_attention_decode_splits) and the splits' fp32 partials are added in split order by a second kernel, so the result
 * is run-to-run deterministic.  A query row with no visible key gets O = 0.  MMB_ERR_UNSUPPORTED when Sq > 16, head_dim
 * is not 64, 96 or 128, or B / H exceed 65535; MMB_ERR_ARG when q, k, v or out is not 16-byte aligned or a stride is not
 * a multiple of 8 elements. */
int mmb_attention_fwd_decode(const void* q, long long ldq, long long bsq, const void* k, long long ldk, long long bsk,
                             const void* v, long long ldv, long long bsv, void* out, long long ldo, long long bso,
                             const void* mask, long long mask_bs, long long mask_qs, int B, int Sq, int Skv, int H,
                             int head_dim, int causal, float scale, void* stream);
/* Number of key splits mmb_attention_fwd_decode uses for (B, H, Skv): a function of its arguments alone (at least 4
 * key blocks of 64 per split, about 264 CTAs, at most 64 splits), >= 1.  Host only. */
int mmb_attention_decode_splits(int B, int H, int Skv);
/* Key / value cache concatenation, torch.cat([past, new], dim=2) of MultiHeadAttentionWithCache
 * (modules/layers/multi_head_attention.py:163-166): past [B, H, Sp, head_dim] (fp32 when past_f32, else bf16; element
 * strides past_bs / past_hs / past_ss, unit stride along head_dim; may be NULL when Sp = 0) and the new projection rows
 * new_rows bf16 [B*Sn, >= H*head_dim] (row stride ld_new) are written as one row-major [B, Sp + Sn, H*head_dim] buffer:
 * out in fp32 (out_f32) or bf16, and / or out_bf16, a bf16 copy (the attention operand when out is fp32).  Either
 * output may be NULL, not both. */
int mmb_kv_cache_append(const void* past, int past_f32, long long past_bs, long long past_hs, long long past_ss,
                        const void* new_rows, long long ld_new, void* out, int out_f32, void* out_bf16, int B, int H,
                        int Sp, int Sn, int head_dim, void* stream);
/* accum[0] += sum_i CE(logits[i,:], labels[i*label_stride]) over rows with label != ignore_index; accum[1] += #rows
 * — nn.CrossEntropyLoss(ignore_index=pad_idx), models/coca/coca_model.py:425,447-450 (forward). */
int mmb_ce_labels(const float* logits, long long ld, const long long* labels, long long label_stride,
                  long long ignore_index, int M, int V, float* row_loss, float* accum, void* stream);

/* ---- contrastive loss -------------------------------------------------------------------------------------- */
/* One direction of contrastive_loss_with_temperature (modules/losses/contrastive_loss_with_temperature.py:81-107),
 * rows = this rank's batch, N = global batch, label(i) = label_offset + i (:39-41).
 * stats: logits = exp(*logit_scale) * sims; row_loss[i] = CE(logits[i], label) with label smoothing; lse_out[i];
 *        *dscale_accum += d(loss_weight * mean_i row_loss)/d logit_scale; optional logits output.
 * grad : dsims (bf16 and/or fp32, leading dim ld_d) = d(loss_weight * sum over ALL ranks of mean row_loss)/d sims of
 *        this rank's row block: the own-direction softmax term plus, for columns [col_lo, col_hi), the transposed
 *        other-direction term rebuilt from the peers' row-LSE vector lse_col[N] — this replaces the reduce-scatter
 *        of torch.distributed.nn.functional.all_gather's backward (utils/distributed.py:47-48).
 *        GLOBAL backprop: [0,N); LOCAL: own block; NONE: lse_col = NULL.
 *  row_w / col_w (optional, NULL = uniform 1/rows): the boolean row `mask` of the reference
 *        (contrastive_loss_with_temperature.py:97-100) as masked-mean weights mask_i / count(mask): row_w[rows] for this
 *        rank's rows, col_w[N] for the global rows (each in its own rank's mean) entering the other-direction term. */
int mmb_contrastive_ce_stats(const float* sims, long long ld, const float* logit_scale, int rows, int N,
                             int label_offset, float label_smoothing, float loss_weight, float* row_loss,
                             float* lse_out, float* dscale_accum, float* logits_out, long long ld_l,
                             const float* row_w, void* stream);
int mmb_contrastive_ce_grad(const float* sims, long long ld, const float* logit_scale, int rows, int N,
                            int label_offset, float label_smoothing, float loss_weight, const float* lse_row,
                            const float* lse_col, int col_lo, int col_hi, void* dsims_bf16, float* dsims_f32,
                            long long ld_d, const float* row_w, const float* col_w, void* stream);
/* fp32 SIMT matmul for tiny / unaligned shapes the tensor-core path rejects: C (+)= alpha*op(A)op(B);
 * ta: A stored [K,M]; tb: B stored [N,K]. */
int mmb_matmul_f32(const float* A, long long lda, int ta, const float* B, long long ldb, int tb, float* C,
                   long long ldc, int M, int N, int K, float alpha, int accumulate, void* stream);
/* out[0] (+)= scale * sum(in[0..n)) — deterministic */
int mmb_sum_scale(const float* in, int n, float scale, float* out, int accumulate, void* stream);


/* ---- GPU input pipeline, image half (SURVEY.md §8 f4) ------------------------------------------------------------- */
/* The CLIP image transform on decoded uint8 RGB images, bit-exact with the reference's PIL / torchvision pipeline
 * (torchmultimodal/transforms/clip_transform.py:300-352: Resize(BICUBIC) + CenterCrop, or RandomResizedCrop with the crop
 * box sampled by the host, then ToTensor + Normalize).  src_ptrs: DEVICE array of n device pointers to HWC uint8 images;
 * geom: DEVICE int32 [n, 12] = {H, W, row pitch (bytes), box_left, box_top, box_w, box_h (the region that is resized, as a
 * standalone image), rw, rh (size it is resized to), crop_left, crop_top (offset of the out x out window in the resized
 * region), flags (bit0: horizontal pass needed = rw != box_w, bit1: vertical pass needed = rh != box_h)};
 * table: DEVICE int32 scratch [n, 2, out, 2 + mmb_clip_image_transform_max_taps()]; outp: fp32 [n, 3, out, out];
 * mean3 / std3: HOST float[3].  The caller guarantees ceil(2 * max(box/r, 1)) * 2 + 1 <= max_taps for both axes. */
int mmb_clip_image_transform_max_taps(void);
int mmb_clip_image_transform(const void* src_ptrs, const int* geom, int* table, float* outp, int n_images, int out,
                             const float* mean3_host, const float* std3_host, void* stream);

/* ---- input pipeline, text half: host-side byte-level BPE (no device work) ------------------------------------------- */
/* The merge loop of CLIPBPETokenizer (torchmultimodal/transforms/clip_transform.py:82-190) as native host code.
 * mmb_bpe_create: merges_utf8 = the whole merges file (header line dropped, then num_merges lines; <= 0: all), bos / eos
 * = the special-token strings; returns an opaque handle and the vocabulary size (512 + merges + 2).
 * mmb_bpe_encode: words = concatenated UTF-8 bytes of the lower-cased, regex-split word pieces of a batch, piece i =
 * [offsets[i], offsets[i+1]); out_ids (capacity offsets[n_words]) receives the ids, out_counts[i] their number per piece.
 * mmb_bpe_token_id: id of a vocabulary string (-1 if absent).  Thread-safe per handle (internal word cache). */
int mmb_bpe_create(const char* merges_utf8, long long n_bytes, int num_merges, const char* bos, const char* eos,
                   void** handle, int* vocab_size);
int mmb_bpe_encode(void* handle, const char* words, const long long* offsets, int n_words, int* out_ids, int* out_counts);
int mmb_bpe_token_id(void* handle, const char* token);
int mmb_bpe_destroy(void* handle);

/* ---- symmetric (CUDA-IPC peer-mapped) memory: the loss path's replacement for NCCL all_gather ----------------- */
/* Replaces torch.distributed(.nn.functional).all_gather at utils/distributed.py:47-52: every rank allocates one
 * buffer, exchanges the 64-byte IPC handles once (host side, any transport), maps the peers' buffers, and the
 * kernels read peer memory directly over NVLink.  handle64 / ptr / peer_ptr are HOST pointers to host variables. */
int mmb_symm_alloc(long long bytes, void** ptr);
int mmb_symm_free(void* ptr);
int mmb_symm_get_handle(void* ptr, void* handle64);
int mmb_symm_open_handle(const void* handle64, void** peer_ptr);
int mmb_symm_close_handle(void* peer_ptr);
/* Cross-GPU barrier on `stream`: release-store `value` into slot [rank] of every peer's flag array, then wait until
 * all `world` slots of my_flags are >= value.  peer_flags is a DEVICE array of `world` device pointers. */
int mmb_symm_signal_wait(void* const* peer_flags, void* my_flags, int rank, int world, int value, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MMB200_H_ */
