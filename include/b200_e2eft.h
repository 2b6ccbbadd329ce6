/* b200_e2eft.h — C ABI of the H100-native single-step denoising engine (libb200_e2eft.so).
 *
 * Drop-in boundary for the hot path named by BASELINE.json `north_star`:
 *   VAE.encode -> UNet2DConditionModel forward (t=999) -> x0 -> VAE.decode.
 * The reference (VisualComputingInstitute/diffusion-e2e-ft) is pure Python and has no FFI of its
 * own; every entry point below replaces the third-party library kernel (cuDNN / cuBLAS / xformers /
 * ATen) behind one leaf operator of the reference's model graph.  The citation after each
 * prototype is the reference call site (relative to the reference repository root) the function serves.
 *
 * Conventions
 *   - plain pointers and sizes only; all pointers are CUDA device pointers owned by the caller
 *     (PyTorch allocates inputs, outputs and workspaces); the library never allocates or syncs;
 *   - kernels are enqueued on `stream` (a cudaStream_t passed as void*);
 *   - return 0 = ok; <0 = invalid argument (nothing launched); >0 = cudaError_t of the launch;
 *     b200_last_error_string() describes the last failure on the calling thread;
 *   - activations are NHWC ("channels last") fp16 operands; the residual stream may be fp16 or fp32
 *     (`*_f32` flags); accumulation, normalisation statistics and softmax are always fp32;
 *   - there is no CPU fallback: without an sm_90a device every launch returns an error.
 */
#ifndef B200_E2EFT_H_
#define B200_E2EFT_H_

#ifdef __cplusplus
extern "C" {
#endif

const char* b200_last_error_string(void);
int b200_abi_version(void);

/* epilogue activations */
#define B200_ACT_NONE 0
#define B200_ACT_SILU 1
#define B200_ACT_GEGLU 2 /* W rows pre-interleaved per tile: [value half | gate half] */
#define B200_ACT_GELU 3  /* erf GELU */
#define B200_ACT_EXP2 4  /* exp2(alpha * acc + bias): softmax probabilities recomputed from the log-sum-exp */

/* out[b][m][n] = act( alpha * sum_k A[b][m][k] * W[(b)][n][k] + bias + residual[b][m][n] )
 * wgmma GEMM, fp16 operands (K contiguous), fp32 accumulate in registers.
 * Replaces: nn.Linear of proj_in/proj_out (GeoWizard/geowizard/models/transformer_2d.py:152-155,
 * 214-217), to_q/to_k/to_v/to_out (attention.py:470-478,501), GEGLU proj + FF out
 * (attention.py:755,765), TimestepEmbedding / time_emb_proj / class_embedding
 * (unet_2d_condition.py:974-1000); batched form = QK^T and PV of the VAE mid attention
 * (unet_2d_blocks.py:589-601). */
int b200_linear(const void* A, long long lda, long long a_batch_stride,
                const void* W, long long ldw, long long w_batch_stride /* 0 = shared */,
                int M, int N, int K, int batch,
                const float* bias, int bias_row,
                const void* residual, long long ld_res, long long res_batch_stride,
                void* out, long long ldo, long long out_batch_stride, int out_f32,
                int act, float alpha,
                double* chan_stats /* optional [M/rows_per_img][N][2]: per-channel sum / sum of squares of
                                      the stored values (caller zeroes): each thread accumulates shifted fp32
                                      partial sums (no cancellation when |mean| >> std) and merges them with
                                      fp64 atomics, so the result is order-independent to ~1e-16 */,
                int rows_per_img,
                void* out2_f16 /* optional fp16 copy of `out` (same strides) for a following GEMM operand */,
                int res_mul /* 1: out = act(alpha*acc + bias) * residual (GEGLU as gate GEMM + value GEMM) */,
                int a_mn /* 1: A is stored [K][M] (row pitch lda >= M): out = A^T-as-stored x W^T without a transposition
                            pass (MN-major wgmma operand).  Weight gradients dW = dY^T X, attention backward dK = dS^T Q */,
                int w_mn /* 1: W is stored [K][N] (row pitch ldw >= N): data gradients dX = dY W, dQ = dS K */,
                long long bias_batch_stride /* bias_row with batch > 1: bias of batch b starts at bias + b * stride */,
                void* stream);

/* GEGLU tile width for packed width N (weights/bias rows are interleaved per tile of this width:
 * [value rows of the tile | gate rows of the tile]); 0 = not tileable. */
int b200_geglu_block_n(int N);

/* Implicit-GEMM convolution on NHWC fp16 input, weights packed [Cout][tap][Cin] (+[C2] shortcut
 * columns), wgmma + TMA, no im2col buffer.  Tap t reads input pixel
 * (ho*stride + tap_dy[t], wo*stride + tap_dx[t]); out-of-range pixels read as zero (padding).
 * Output pixel (ho,wo) is written at (ho*out_mul+out_oy, wo*out_mul+out_ox) of an
 * (Ho*out_mul x Wo*out_mul) NHWC (or NCHW when out_nchw) tensor.
 *   out = act( conv(X) + conv1x1(X2) + bias[c] + rowvec[img][c] + residual )
 * Replaces: ResnetBlock2D.conv1/conv2/conv_shortcut (instantiated at
 * GeoWizard/geowizard/models/unet_2d_blocks.py:1064-1076,1211-1223,2242-2254,2400-2412,667-679),
 * Downsample2D.conv (:1107-1113,1228-1234, VAE :1315-1321), Upsample2D.conv (:2285,2417),
 * conv_out (unet_2d_condition.py:617-619) and the VAE encoder/decoder convs
 * (Marigold/marigold/marigold_pipeline.py:493,516). */
int b200_conv2d_nhwc(const void* X, int NB, int H, int W, int Cin,
                     const void* X2, int C2,
                     const void* Wp, int Cout, int num_taps, const int* tap_dy, const int* tap_dx,
                     int stride, int Ho, int Wo, int out_mul, int out_oy, int out_ox,
                     const float* bias, const float* rowvec, long long ld_rowvec,
                     const void* residual, void* out, int out_f32, int out_nchw, int act,
                     double* chan_stats /* optional [NB][Cout][2], see b200_linear */,
                     void* out2_f16 /* optional fp16 NHWC copy of `out` */, void* stream);

/* 3x3 / stride 1 / pad 1 convolution with Cout <= 8 (the `conv_out` layers: unet_2d_condition.py:617-619
 * and the VAE encoder/decoder conv_out): NHWC fp16 in (C % 64 == 0), NCHW fp32 out, input read once.
 * wq: fp16 [C/64][9 taps][4 k-steps][8 n][16 k] (zero padded to 8 output channels). */
int b200_conv3x3_small_cout(const void* x, int NB, int H, int W, int C, const void* wq,
                            const float* bias, int Cout, float* out, void* stream);

/* Patch matrix for the small-Cin input convolutions (conv_in: 8->320, 3->128, 4->512):
 * out[pixel][tap*Cin + c] fp16, row length Kpad (zero padded).  `x` is NCHW (x_f32 ? fp32 : fp16).
 * Serves unet_2d_condition.py:294-296,1084 and the VAE conv_in. */
int b200_im2col3x3_nchw(const void* x, int x_f32, int NB, int C, int H, int W, void* out,
                        int Kpad, void* stream);

/* GroupNorm statistics over NHWC input that is the channel-concatenation of up to two tensors
 * (skip-connection concat, unet_2d_blocks.py:2328,2456, is never materialised).
 * sums[n][g][2] (double) must be zeroed by the caller. */
int b200_group_norm_stats(const void* x1, int C1, const void* x2, int C2, int in_f32, int NB,
                          int HW, int groups, double* sums, void* stream);
/* y = [silu]( (x-mean)*rstd*gamma + beta ) as fp16 NHWC; optional raw fp16 copy of the
 * (concatenated) input for the 1x1 shortcut operand.
 * Replaces GroupNorm+SiLU of ResnetBlock2D norm1/norm2, conv_norm_out
 * (unet_2d_condition.py:605-610,1209-1211) and Transformer2DModel.norm (transformer_2d.py:151,331). */
int b200_group_norm_apply(const void* x1, int C1, const void* x2, int C2, int in_f32, int NB, int HW,
                          int groups, const double* sums, const float* gamma, const float* beta,
                          float eps, int silu, void* y, void* raw_copy, void* stream);

/* Same, but the statistics come from per-channel sums produced by the epilogue of the kernel that wrote
 * each source (chan_stats of b200_linear / b200_conv2d_nhwc): cs1 [NB][C1][2], cs2 [NB][C2][2] (fp64). */
int b200_group_norm_apply_cs(const void* x1, int C1, const double* cs1, const void* x2, int C2,
                             const double* cs2, int in_f32, int NB, int HW, int groups,
                             const float* gamma, const float* beta, float eps, int silu, void* y,
                             void* raw_copy, void* stream);

/* LayerNorm over the last dim of [rows][C] (in_f32 ? fp32 : fp16) -> fp16.
 * Replaces BasicTransformerBlock.norm1/2/3 (attention.py:205,237,264). */
int b200_layer_norm(const void* x, int in_f32, long long rows, int C, const float* gamma,
                    const float* beta, float eps, void* y, void* stream);

/* Flash attention over heads of width head_dim in {40, 64, 80, 160} (ABI 14; any other width returns a negative
 * code before launch), fp16 Q/K/V read in place from (possibly fused) projection buffers: element (b, l, h, d) of Q
 * is q[b*q_bs + l*q_ls + h*head_dim + d] (same for K, V).  head_dim 40 / 80 / 160 are the SD-1.x UNet's 320 / 640 /
 * 1280 channels over 8 heads (GeoWizard); 64 is SD-2's.
 * `kv_segments` = 2 implements GeoWizard's joint self-attention: batch element b attends to the
 * keys/values of b%(B/2) and b%(B/2)+B/2 concatenated (attention.py:482-491).
 * out[b][l][h*head_dim+d] fp16 with row stride o_ls.   softmax(QK^T*scale)V, fp32 softmax.
 * Strides are multiples of 8 elements, pointers 16-byte aligned, 1 <= B, heads <= 65535.
 * Replaces xformers.ops.memory_efficient_attention (attention.py:497) / attn1, attn2
 * (attention.py:338-343,375-380). */
int b200_attention(const void* q, long long q_bs, long long q_ls,
                   const void* k, long long k_bs, long long k_ls,
                   const void* v, long long v_bs, long long v_ls,
                   void* out, long long o_bs, long long o_ls,
                   int B, int heads, int head_dim, int Lq, int Lk, int kv_segments, float scale,
                   float* lse /* optional [B][heads][Lq] fp32: log2-domain log-sum-exp of the scaled scores, so that
                                 P_ij = exp2(scale * log2(e) * S_ij - lse_i) — the backward pass recomputes P from it */,
                   void* stream);
/* b200_attention with head_dim = 64. */
int b200_attention_d64(const void* q, long long q_bs, long long q_ls,
                       const void* k, long long k_bs, long long k_ls,
                       const void* v, long long v_bs, long long v_ls,
                       void* out, long long o_bs, long long o_ls,
                       int B, int heads, int Lq, int Lk, int kv_segments, float scale, float* lse, void* stream);

/* Flash attention, one head of width 512 (the VAE mid-block), fp16 Q/K/V read in place from a
 * (possibly fused) projection buffer: element (b, l, d) of Q is q[b*q_bs + l*q_ls + d] (same for K, V).
 * out[b][l][d] = out[b*o_bs + l*o_ls + d] fp16.  softmax(QK^T*scale)V with fp32 scores and softmax
 * statistics, fp16 P, fp32 accumulation; the L x L score matrix is never stored, so memory is O(L).
 * Strides are multiples of 8 elements, row strides >= 512, pointers 16-byte aligned, 1 <= B <= 65535,
 * Lq, Lk >= 1 (ragged lengths are fine).  No log-sum-exp output and no backward counterpart.
 * Replaces the memory-efficient (xformers) attention of the VAE mid-block: unet_2d_blocks.py:589-601
 * with `enable_xformers_memory_efficient_attention` (Marigold/run.py:285). */
int b200_attention_d512(const void* q, long long q_bs, long long q_ls,
                        const void* k, long long k_bs, long long k_ls,
                        const void* v, long long v_bs, long long v_ls,
                        void* out, long long o_bs, long long o_ls,
                        int B, int Lq, int Lk, float scale, void* stream);

/* Row softmax: P[r][:] = softmax(scale * S[r][:]) fp32 -> fp16 (VAE mid-block attention, d=512). */
int b200_softmax_rows(const float* S, long long lds, void* P, long long ldp, long long rows,
                      int cols, float scale, void* stream);

/* Grouped softmax for the constant-context cross-attention specialisation (SURVEY.md §8 f1;
 * Marigold/marigold/marigold_pipeline.py:428-432 repeats ONE [1,2,1024] empty-text embedding over the batch,
 * GeoWizard/geowizard/models/attention.py:375-380 attends to it): logits [rows][ld_in] fp32, column
 * head*S + s; softmax over the S keys of every head -> fp16 [rows][ld_out] (columns >= heads*S zeroed). */
int b200_softmax_groups(const float* logits, int ld_in, long long rows, int heads, int S, void* P, int ld_out,
                        void* stream);

/* Nearest-neighbour resize NHWC (in_f32 ? fp32 : fp16) -> fp16 (Upsample2D interpolate,
 * exact 2x or explicit `size=`, unet_2d_condition.py:1185-1186). */
int b200_upsample_nearest_nhwc(const void* x, int in_f32, int NB, int H, int W, int C, int OH,
                               int OW, void* y, void* stream);

/* Sinusoidal timestep embedding (flip_sin_to_cos, freq_shift 0) -> fp16 [B][dim].
 * t is a device array of B floats.  unet_2d_condition.py:974. */
int b200_timestep_embedding(const float* t, int B, int dim, void* out, void* stream);

/* CLIP text embeddings: out[r][c] = tok[ids[r]][c] + pos[r % L][c], fp32 [rows][C]; ids int64 (clamped to the table);
 * tables fp16 or fp32 (w_f32).  transformers==4.37.2 models/clip/modeling_clip.py CLIPTextEmbeddings.forward, reached
 * from Marigold/marigold/marigold_pipeline.py:369 (`self.text_encoder(text_input_ids)[0]`). */
int b200_embed_tokens(const long long* ids, const void* tok, const void* pos, int w_f32, long long rows, int L, int C,
                      int vocab, float* out, void* stream);

/* Small dense per-pixel channel mix on NCHW fp32 (Cin, Cout <= 8):
 * out[n][co][p] = sum_ci Wm[co][ci] * (a1*in1[n][ci][p] + a2*in2[n][ci][p]) + bias[co].
 * Serves quant_conv + latent scaling (marigold_pipeline.py:494-497) and
 * pred_original_sample + /0.18215 + post_quant_conv (:457-465,513-515). */
int b200_pointwise_nchw(const float* in1, float a1, const float* in2, float a2, int in_cstride,
                        const float* Wm, const float* bias, int NB, int Cin, int Cout, long long HW,
                        float* out, void* stream);

/* One DDIM update (diffusers DDIMScheduler.step, eta = 0) on NCHW latents, fp32 arithmetic in diffusers' order:
 *   beta = 1 - a_t;  x0, eps from the prediction type:
 *     B200_PRED_V:       x0 = sqrt(a_t) x - sqrt(beta) m,   eps = sqrt(a_t) m + sqrt(beta) x
 *     B200_PRED_EPSILON: x0 = (x - sqrt(beta) m) / sqrt(a_t), eps = m
 *     B200_PRED_SAMPLE:  x0 = m,                            eps = (x - sqrt(a_t) x0) / sqrt(beta)
 *   prev = sqrt(a_prev) x0 + sqrt(1 - a_prev) eps.
 * model_out m: [B][C][HW] (mo_f16 ? fp16 : fp32), batch stride mo_bstride; sample x: fp32, batch stride s_bstride,
 * NULL = exact zeros.  prev_sample: fp32 [B][C][HW] contiguous, may alias sample (then s_bstride = C*HW);
 * pred_original_sample: fp32 [B][C][HW] or NULL.  unet_in (nullable): prev cast to fp16 (unet_in_f16) or fp32, written
 * at unet_in[b*ui_bstride + c*HW + p] -- the noisy-latent channel slice of the next step's UNet input, so the
 * per-step concatenation and cast disappear.  0 < a_t < 1, 0 <= a_prev <= 1.
 * Replaces scheduler.step at Marigold/marigold/marigold_pipeline.py:457-465 and
 * GeoWizard/geowizard/models/geowizard_pipeline.py:326-334. */
#define B200_PRED_EPSILON 0
#define B200_PRED_V 1
#define B200_PRED_SAMPLE 2
int b200_ddim_step(const void* model_out, int mo_f16, long long mo_bstride, const float* sample, long long s_bstride,
                   int B, int C, long long HW, int prediction_type, float alpha_prod_t, float alpha_prod_t_prev,
                   float* prev_sample, float* pred_original_sample, void* unet_in, int unet_in_f16,
                   long long ui_bstride, void* stream);

/* Decode post-ops on NCHW fp32 [B][3][HW]: mode 0 = depth: (clip(mean_c, -1, 1)+1)/2 -> [B][1][HW];
 * mode 1 = normals: x/(||x||_2+1e-5) * sign -> [B][3][HW] (marigold_pipeline.py:467-478);
 * mode 2 / 3 = the training variants: clip(mean_c) without the affine map / normalised then clamped
 * (training/train.py:532-540). */
int b200_decode_post(const float* x, int NB, long long HW, int mode, float sign, float* out,
                     void* stream);

/* Task losses of the E2E fine-tuning step, forward only (training/util/loss.py:13-67, training/train.py:542-556).
 * pred/target NCHW fp32 ([B][1][HW] depth, [B][3][HW] normals), mask [B][HW] bytes, workspace: zeroed doubles
 * (5*B + 2 for SSI, 2 for angular), out: one float (mean over masked pixels; nan for an empty mask). */
int b200_ssi_loss(const float* pred, const float* target, const unsigned char* mask, int B, long long HW,
                  double* workspace, float* out, void* stream);
int b200_angular_loss(const float* pred, const float* target, const unsigned char* mask, int B, long long HW,
                      double* workspace, float* out, void* stream);

/* Optimizer side of the fine-tuning step on flat fp32 buffers (training/train.py:346-353,564-566):
 * sum of squares (gradient norm; `out` is a zeroed double accumulated with atomics) and a fused
 * clip_grad_norm_ + torch.optim.AdamW update (decoupled weight decay, bias correction by `step` >= 1).
 * grad_norm_sq (device, may be NULL) and max_grad_norm give the clip coefficient without a host sync. */
int b200_sumsq(const float* x, long long n, double* out, void* stream);
int b200_adamw_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                    float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                    const double* grad_norm_sq, float max_grad_norm, void* stream);
/* Same with a loss-scaled gradient buffer: grad holds S*g and grad_norm_sq = |S*g|^2; grad_unscale = 1/S. */
int b200_adamw_step_scaled(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                           float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                           const double* grad_norm_sq, float max_grad_norm, float grad_unscale, void* stream);

/* Same update driven by a device-side state block (fp32[8]: loss scale, growth tracker, applied steps, skipped
 * steps, skipped flag, gradient multiplier, bc1, bc2) so that neither the skip decision nor dynamic loss scaling
 * needs a host sync: the step is skipped (parameters and moments untouched, as torch.optim.AdamW leaves parameters
 * whose .grad is None) when the gradient norm is non-finite (fp16 overflow of the loss-scaled backward: the scale is
 * halved) or exactly zero (empty validity masks / NaN loss: training/train.py:503,546-551 back-propagates 0).
 * `grad` holds (loss scale x world size) x the mean gradient; inv_world = 1 / data-parallel ranks. */
int b200_adamw_step_state(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                          float lr, float beta1, float beta2, float eps, float weight_decay,
                          const double* grad_norm_sq, float max_grad_norm, float inv_world, float* state,
                          int dynamic_scale, float growth_interval, float min_scale, float max_scale, void* stream);

/* Per-group learning rates (ABI 11): torch.optim.AdamW with parameter groups, e.g. GeoWizard's two groups of
 * train_depth_normal.py:428-444 (every `class_embedding.*` parameter at learning_rate * class_embedding_lr_mult) or
 * Marigold's one group of training/train.py:346-353.  The flat buffer is cut into n_runs RUNS: run r covers elements
 * [run_start[r], run_start[r+1]) (the last one up to n) and belongs to group run_group[r]; run_start (int64) and
 * run_group (int32) live on the DEVICE, run_start[0] == 0, starts increase and are multiples of 4.  group_lr /
 * group_wd are HOST arrays of n_groups values, passed with the launch.  With n_runs == 1 the tables may be NULL (the
 * whole buffer is group 0).  Everything else, the state block and its single skip decision / loss scale / bias
 * correction included, is b200_adamw_step_state's (which is this call with one run).  Per element the arithmetic is
 * unchanged: decay = 1 - lr*wd, step_size = lr / bc1 of the element's group. */
#define B200_ADAMW_MAX_GROUPS 16
#define B200_ADAMW_MAX_RUNS 1024
int b200_adamw_step_state_groups(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                                 const long long* run_start, const int* run_group, int n_runs, const float* group_lr,
                                 const float* group_wd, int n_groups, float beta1, float beta2, float eps,
                                 const double* grad_norm_sq, float max_grad_norm, float inv_world, float* state,
                                 int dynamic_scale, float growth_interval, float min_scale, float max_scale,
                                 void* stream);

/* ---- Backward pass (training/train.py:545-566, `accelerator.backward(loss)`).  The GEMM-shaped halves run on
 * b200_linear / b200_conv2d_nhwc with re-packed operands; these are the streaming / reduction kernels around them.
 *
 * b200_gather_planar: out[c][q] (fp16, row stride ldo >= NB*Ho*Wo, zero-filled past the last pixel) =
 *   x[n][(stride*o + oy)/up][(stride*p + ox)/up][c] (pixel stride ldx >= C) with q = (n*Ho + o)*Wo + p, zero outside the (up-sampled)
 *   image: the K-major (K = pixels) operand of a weight-gradient GEMM for one kernel tap of a stride-1/-2 or
 *   nearest-2x-upsampled 3x3 conv; with Ho=H, Wo=W, stride=1, up=1, oy=ox=0 a plain [rows][C] -> [C][rows] transpose.
 * b200_col_sum: out[c] += sum_rows x[row][c] (bias gradients).
 * GroupNorm backward (diffusers GroupNorm(32) + optional SiLU, NHWC): mean_rstd [NB][groups][2] from the
 *   forward's statistics; pass 1 accumulates S [NB][Ctot][2] = (sum dz, sum dz*xhat) per channel (zeroed by
 *   the caller; call once per concatenated input with its channel offset), pass 2 writes
 *   dx = rstd*(dz*gamma - mean_g(gamma dz) - xhat*mean_g(gamma dz xhat)) (+ add).  d_gamma = sum_n S[..1],
 *   d_beta = sum_n S[..0].  dy is fp16 [NB][HW][Ctot].
 * b200_layer_norm_bwd: dx (+ add) and d_gamma/d_beta (accumulated into zeroed fp32 [C]).
 * b200_softmax_bwd_rows: dS = scale * P o (dP - rowsum(dP o P)), P/dS fp16, dP fp32.
 * b200_act_bwd: dx = dy * act'(x), act = B200_ACT_SILU | B200_ACT_GELU (fp16).
 * b200_geglu_bwd: y = h*gelu(g): dh = dy*gelu(g), dg = dy*h*gelu'(g). */
int b200_gather_planar(const void* x, int in_f32, long long ldx, int NB, int H, int W, int C, int Ho, int Wo, int stride, int up,
                       int oy, int ox, void* out, long long ldo, void* stream);
int b200_col_sum(const void* x, int in_f32, long long rows, int C, long long ld, float* out, void* stream);
/* delta[b][h][t] = sum_d a[b,t,h*D+d] * c[b,t,h*D+d] (fp16 in, fp32 out), D = head_dim in {40, 64, 80, 160} (ABI 14):
 * the row term of the softmax backward, dS = scale * P o (dP - delta), with a = dO and c = O (attention backward,
 * attention.py:497).  b200_rowdot_heads is the head_dim = 64 call. */
int b200_rowdot_heads_d(const void* a, long long a_bs, long long a_ls, const void* c, long long c_bs, long long c_ls,
                        int B, int L, int heads, int head_dim, float* out, void* stream);
int b200_rowdot_heads(const void* a, long long a_bs, long long a_ls, const void* c, long long c_bs, long long c_ls,
                      int B, int L, int heads, float* out, void* stream);
int b200_group_norm_mean_rstd(const double* sums, const double* cs1, int C1, const double* cs2, int C2, int NB, int HW,
                              int groups, float eps, float* mean_rstd, void* stream);
int b200_group_norm_bwd_sums(const void* x, int in_f32, int Cx, int c_off, int Ctot, const void* dy, int NB, int HW,
                             int groups, const float* mean_rstd, const float* gamma, const float* beta, int silu,
                             float* S, void* stream);
int b200_group_norm_bwd_apply(const void* x, int in_f32, int Cx, int c_off, int Ctot, const void* dy, int NB, int HW,
                              int groups, const float* mean_rstd, const float* gamma, const float* beta, int silu,
                              const float* S, const void* add, void* dx, int out_f32, void* stream);
int b200_layer_norm_bwd(const void* x, int in_f32, long long rows, int C, const float* gamma, const void* dy,
                        float eps, const void* add, void* dx, int out_f32, float* dgamma, float* dbeta, void* stream);
int b200_softmax_bwd_rows(const void* P, long long ldp, const float* dP, long long ldd, void* dS, long long rows,
                          int cols, float scale, void* stream);
int b200_act_bwd(const void* x, const void* dy, long long n, int act, void* dx, void* stream);
int b200_geglu_bwd(const void* h, const void* g, long long ld_hg, const void* dy, long long rows, int inner, void* dh,
                   void* dg, long long ld_d, void* stream);

/* Loss / post-op backward of the fine-tuning step (training/train.py:532-556, training/util/loss.py):
 * d(loss)/d(pred) * grad_out[0] (device scalar: the upstream gradient, i.e. the loss scale).  The SSI gradient
 * flows through the per-image least-squares scale/shift, as torch.autograd does in the reference.
 * workspace: zeroed doubles, 7*B (ssi) / 1 (angular).  decode_post_bwd: modes 2 (depth) / 3 (normals). */
int b200_ssi_loss_bwd(const float* pred, const float* target, const unsigned char* mask, int B, long long HW,
                      double* workspace, const float* grad_out, float* dpred, void* stream);
int b200_angular_loss_bwd(const float* pred, const float* target, const unsigned char* mask, int B, long long HW,
                          double* workspace, const float* grad_out, float* dpred, void* stream);
int b200_decode_post_bwd(const float* x, const float* dout, int NB, long long HW, int mode, float* dx, void* stream);
/* Backward of b200_upsample_nearest_nhwc (explicit output size, unet_2d_condition.py:1185-1186): fp32 NHWC,
 * dx[n,h,w,:] = (add) + sum of dy over the output pixels whose nearest source is (h,w). */
int b200_upsample_nearest_bwd(const float* dy, int NB, int H, int W, int C, int OH, int OW, const float* add,
                              float* dx, void* stream);

/* fp32 <-> fp16 casts / layout helpers used at module boundaries. */
int b200_cast_f32_to_f16(const float* x, void* y, long long n, void* stream);
int b200_nhwc_to_nchw_f32(const void* x, int in_f32, int NB, int C, long long HW, float* y, void* stream);

/* debugging: force a BLOCK_N (0 = automatic) */
void b200_debug_force_block_n(int bn);
/* debugging / perf experiments (results are wrong when set): 1 = skip epilogue stores, 2 = skip A loads,
 * 4 = skip W loads */
void b200_debug_set_flags(int flags);
/* 1 (default) = swap operands automatically when Cout % 128 == 0; 0 = never */
void b200_debug_set_swap(int mode);
void b200_debug_set_halo(int mode);   /* 1 = automatic halo-resident stride-1 3x3 conv (default), 0 = per-tap boxes */
int b200_debug_last_path(void);       /* path of the last b200_conv2d_nhwc call: 1 = halo-resident, 0 = per-tap boxes */
/* Record of the last gemm_conv_kernel launch, from b200_linear or b200_conv2d_nhwc (ABI 12): which template instantiation
 * ran and on which tile geometry.  Copies min(n, 16) ints to out and returns 16 (the record length; out may be NULL).
 * Fields: 0 conv (1) / linear (0), 1 halo-resident, 2 swapped orientation, 3 BLOCK_N, 4 vectorised epilogue (VEC),
 * 5 GEGLU, 6 fp32 output, 7 bw, 8 bh, 9 halo_n (halo MMA width), 10 tiles_w, 11 tiles_h, 12 m_tiles, 13 n_tiles,
 * 14 grid (CTAs), 15 fused statistics.  Debug only: nothing on the launch path reads it. */
int b200_debug_last_launch(int* out, int n);

/* torchvision resize(x, size, BICUBIC, antialias=True) of [planes][H][W] fp32 (aten _upsample_bicubic2d_aa, Keys
 * cubic a = -0.5): the CLIP image-encoder input of GeoWizard/geowizard/models/geowizard_pipeline.py:239-243.
 * tmp: [planes][H][OW] fp32 scratch. */
int b200_resize_bicubic_aa(const float* x, long long planes, int H, int W, int OH, int OW, float* tmp, float* out,
                           void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Host-pipeline post/pre-processing on the device (SURVEY.md §8 a11, f2).
 *
 * b200_ensemble_normals: Marigold/marigold/marigold_pipeline.py:59-71 == GeoWizard/geowizard/utils/
 *   normal_ensemble.py:6-22.  preds [E][3][HW] fp32 (E <= 32) -> out [3][HW] = preds[index] / (|.| + 1e-5) with
 *   index = argmin_e sum_pixels acos(clip(cos(mean-angle normal, n_e), +-0.999)); err_ws = double[E] scratch.
 * b200_ensemble_depths_objective / _reduce: Marigold/marigold/util/ensemble.py:40-132.  imgs [E][HW] fp32, s/t [E]
 *   device fp32.  objective: ws (double[2] scratch) [0] = sum over pixels and pairs i<j of (v_i - v_j)^2,
 *   out3[1], out3[2] = min / max of the reduced map (the scipy-BFGS closure :74-98 finishes on the host);
 *   reduce: aligned / uncertainty [HW] = median + MAD (reduction 0) or mean + std (1), scaled to [0, 1] (:110-130).
 * b200_minmax_rows: per-row (min, max) of [rows][cols] fp32 -> out[rows][2] (ws: uint32[2*rows]) (:66-69 init guess).
 * b200_minmax_normalise: x = (x - min x) / (max x - min x) in place (marigold_pipeline.py:305-312); minmax_out[2] opt.
 * b200_rgb_normalise: uint8 / fp32 [0,255] -> fp32 x / 255 * 2 - 1 (:245-247).
 * b200_resize_bilinear_aa: torchvision resize(..., BILINEAR, antialias=True) of [planes][H][W] fp32 (:237-242,315-321),
 *   separable (width then height), tmp = [planes][H][OW] scratch.   b200_resize_nearest: geowizard normals. */
int b200_ensemble_normals(const float* preds, int E, long long HW, double* err_ws, float* out, int* index, void* stream);
int b200_ensemble_depths_objective(const float* imgs, const float* s, const float* t, int E, long long HW,
                                   int reduction, double* ws, float* out3, void* stream);
int b200_ensemble_depths_reduce(const float* imgs, const float* s, const float* t, int E, long long HW, int reduction,
                                double* ws, float* aligned, float* uncertainty, void* stream);
int b200_minmax_rows(const float* x, int rows, long long cols, unsigned int* ws, float* out, void* stream);
int b200_minmax_normalise(float* x, long long n, unsigned int* ws, float* minmax_out, void* stream);
int b200_rgb_normalise(const void* x, int in_u8, long long n, int round_u8, float* out, void* stream);
int b200_resize_bilinear_aa(const float* x, long long planes, int H, int W, int OH, int OW, float* tmp, float* out,
                            void* stream);
int b200_resize_nearest(const float* x, long long planes, int H, int W, int OH, int OW, float* out, void* stream);

/* Resampling choice and colour outputs of the pipelines' __call__ (ABI 9).
 * b200_resize_nearest_exact: torch interpolate(mode="nearest-exact") of [planes][H][W] fp32 -> [planes][OH][OW],
 *   src = min(floor((dst + 0.5) * (in / out)), in - 1) with the fp32 scale; the reference's resample_method="nearest"
 *   (Marigold/marigold/util/image_util.py:111-116, marigold_pipeline.py:219,237-242,315-321).
 * b200_colorize_depth: fp32 [n] -> uint8 [n][3] through table [ncol][3] uint8 (ncol <= 4096):
 *   colorize_depth_maps(pred, 0, 1, cmap) then (colored * 255).astype(uint8) and chw2hwc
 *   (Marigold/marigold/util/image_util.py:29-67, marigold_pipeline.py:327-338, geowizard_pipeline.py:211-216);
 *   index (int)(clip(x, 0, 1) * ncol) with ncol -> ncol - 1, NaN -> (0, 0, 0); out 4-byte aligned.
 * b200_colorize_normals: fp32 [3][HW] -> uint8 [HW][3] = ((clip(x, -1, 1) + 1) / 2 * 255) truncated, NaN -> 0
 *   (marigold_pipeline.py:339-343, geowizard_pipeline.py:218-219); out 4-byte aligned. */
int b200_resize_nearest_exact(const float* x, long long planes, int H, int W, int OH, int OW, float* out, void* stream);
int b200_colorize_depth(const float* x, long long n, const unsigned char* table, int ncol, unsigned char* out,
                        void* stream);
int b200_colorize_normals(const float* x, long long HW, unsigned char* out, void* stream);

/* Diffusion-objective training and the EMA of the UNet weights (ABI 10).
 * b200_diffusion_inputs: DDPMScheduler.add_noise + get_velocity + the UNet-input concatenation of
 *   GeoWizard/geowizard/training/train_depth_normal.py:666-705 (the default, non-`--e2e_ft` branch) in one pass.
 *   rgb_latents [B][C][HW], x0 / noise [2B][C][HW] (depth half, then normal half; noise NULL = zeros), timesteps int64
 *   [2B] and alphas_cumprod fp32 [T] on the device (0 <= t < T, checked by the caller), all fp32.  With a = ac[t[n]]:
 *     unet_in [2B][2C][HW] = [rgb[n mod B] | sqrt(a) x0 + sqrt(1 - a) eps],
 *     target  [2B][C][HW]  = eps (B200_PRED_EPSILON) or sqrt(a) eps - sqrt(1 - a) x0 (B200_PRED_V),
 *   each product and sum rounded on its own: bit-identical to torch's fp32 evaluation of diffusers' expressions.
 * b200_masked_latent_mse: F.mse_loss(pred[latent_mask], target[latent_mask]) of :607-609,712-714 with
 *   latent_mask = ~max_pool2d(~val_mask, 8, 8) repeated over the 2 halves and C channels.  pred [2B][C][h][w]
 *   (pred_f16 ? fp16 : fp32), target fp32, val_mask [B][H][W] bytes with h = H / 8, w = W / 8.  Writes latent_mask
 *   [B][h][w] bytes (for the backward), workspace (2 zeroed doubles: fp64 sum of squares, exact count) and out[0] =
 *   sum / count, 0 for an empty mask.  No host sync.
 * b200_masked_latent_mse_bwd: grad = grad_out[0] * 2 (pred - target) / count on the latent mask, 0 elsewhere, in
 *   pred's dtype and layout; latent_mask and workspace are the forward's.
 * b200_ema_update: diffusers EMAModel.step (train_depth_normal.py:351-353,785-786) over flat fp32 buffers:
 *   ema <- ema - one_minus_decay * (ema - param), each operation rounded on its own; 16-byte aligned buffers. */
int b200_diffusion_inputs(const float* rgb_latents, const float* x0, const float* noise, const long long* timesteps,
                          const float* alphas_cumprod, int B, int C, long long HW, int prediction_type, float* unet_in,
                          float* target, void* stream);
int b200_masked_latent_mse(const void* pred, int pred_f16, const float* target, const unsigned char* val_mask, int B,
                           int C, int H, int W, int h, int w, unsigned char* latent_mask, double* workspace, float* out,
                           void* stream);
int b200_masked_latent_mse_bwd(const void* pred, int pred_f16, const float* target, const unsigned char* latent_mask,
                               const double* workspace, const float* grad_out, int B, int C, long long hw, void* grad,
                               void* stream);
int b200_ema_update(float* ema, const float* param, long long n, float one_minus_decay, void* stream);

/* Evaluation of depth and normal predictions (ABI 13).  Every sum is an fp64 partial per block, combined in a fixed
 * order (no floating-point atomics: two runs give the same bits); counts and indices are 64-bit; nothing syncs the
 * host.  Maps are fp32, masks bytes (nonzero = valid), all on the device.  `ws` workspaces hold
 * B x B200_EVAL_MAX_BLOCKS x (7 | 11 | 8) doubles for align_depth / depth_metrics / normal_error.
 *
 * b200_eval_align_depth: Marigold/src/util/alignment.py:8-55 (np.linalg.lstsq of [p 1] x = g over the mask) as called
 *   at Marigold/eval.py:173-203.  gt / pred / mask [B][H][W].  The moments are taken over every row and the columns
 *   j < OW at source column min(floor(float(j) * col_scale), W - 1): the grid torch.nn.Upsample(scale_factor=s,
 *   mode="nearest") samples from the [1, H, W] tensor of alignment.py:26 (OW = floor(W * s), col_scale = float(1 / s);
 *   OW = W for no down-sampling).  disparity: the target is 1 / gt and the mask is mask & gt > 0 & pred > 0
 *   (eval.py:182-197).  scale_shift [B][2] fp32 from a 2x2 solve in fp64; a constant prediction p gets lstsq's
 *   minimum-norm solution (p, 1) * mean(g) / (p^2 + 1), an empty mask (0, 0).
 * b200_eval_depth_metrics: eval.py:173-220 after the solve, one pass over pred / gt / mask [B][HW] (mask NULL = the
 *   metrics' valid_mask=None):  p = pred * s + t (two fp32 roundings, scale_shift NULL = no alignment); disparity:
 *   p = 1 / max(p, 1e-3); clip: p = max(clip(p, min_depth, max_depth), 1e-6).  aligned (nullable) [B][HW] receives p.
 *   out (nullable: then gt may be NULL and only `aligned` is written) fp32[10] = abs_relative_difference,
 *   squared_relative_difference, rmse_linear, rmse_log, log10, delta1_acc, delta2_acc, delta3_acc, i_rmse, silog_rmse
 *   of Marigold/src/util/metric.py with its batch semantics: per-sample means averaged over B, log10 pooled over the
 *   batch's pixels, silog with the batch mean inside the sqrt.  Per-pixel terms fp32, sums fp64; an empty mask gives NaN.
 * b200_eval_normal_error: DSINE/utils/utils.py:150-159 and the accumulation of DSINE/projects/dsine/test.py:100-115.
 *   pred / gt [B][3][H][W] read with element strides {b, c, h, w} (host arrays), so [3,H,W] and [H,W,3] maps are read in
 *   place; mask [B][H][W] (NULL = every pixel).  Angle acos(clamp(x.y / (max(|x|,1e-8) max(|y|,1e-8)), -1, 1)) * 180 / pi
 *   in degrees (torch.cosine_similarity), the cosine in fp64 rounded once to fp32.  err_map (nullable) [B][H][W].  buf (nullable): the
 *   masked angles are appended, compacted in no particular order, at buf[*buf_len ...] (*buf_len advanced; writes past
 *   buf_capacity are dropped).  sums / counts (nullable together): sums[2] += (sum e, sum e^2), counts[6] += (n, #e < 5,
 *   7.5, 11.25, 22.5, 30) over the masked pixels.
 * b200_eval_kth_smallest: exact k-th smallest (0-based) of x[0 .. *n) (*n read on the device; n_max >= *n sizes the
 *   grid) by a radix select on the fp32 bit patterns: finite, non-negative values (-0 counts as +0).  k < 0 = the
 *   median: k = (n - 1) / 2.  out[0] = k-th, out[1] = (k+1)-th (the k-th when k is the last), out[2] = the median as
 *   np.median gives it on a float32 array ((out[0] + out[1]) / 2 in fp32 for an even count) for k < 0, out[0] else;
 *   NaN when k >= n.  ws: unsigned long long[B200_EVAL_KTH_WS_WORDS]. */
#define B200_EVAL_MAX_BLOCKS 512
#define B200_EVAL_KTH_WS_WORDS 261
int b200_eval_align_depth(const float* gt, const float* pred, const unsigned char* mask, int B, int H, int W, int OW,
                          float col_scale, int disparity, double* ws, float* scale_shift, void* stream);
int b200_eval_depth_metrics(const float* pred, const float* gt, const unsigned char* mask, int B, long long HW,
                            const float* scale_shift, int disparity, int clip, float min_depth, float max_depth,
                            float* aligned, double* ws, float* out, void* stream);
int b200_eval_normal_error(const float* pred, const long long* pred_strides, const float* gt,
                           const long long* gt_strides, const unsigned char* mask, int B, int H, int W, float* err_map,
                           float* buf, long long buf_capacity, unsigned long long* buf_len, double* ws, double* sums,
                           long long* counts, void* stream);
int b200_eval_kth_smallest(const float* x, const unsigned long long* n, long long n_max, long long k,
                           unsigned long long* ws, float* out, void* stream);

/* Training-batch preparation (ABI 15): the per-sample transforms of training/dataloaders/load.py on decoded images,
 * bitwise as the reference computes them.  Images are uint8 [B][H][W][3] (HWC), depths uint16 [B][H][W]; flip
 * (nullable = no sample flipped) is one byte per sample, nonzero = horizontally flipped.  Nothing syncs the host.
 *
 * b200_data_hypersim_source: depth_m = float32(mm / 1000.0); the normals re-oriented towards the camera as
 *   Hypersim.align_normals does in fp64 (inv_k: the 3x3 inverse intrinsics, row-major, on the host) and re-quantised
 *   to uint8 by truncation; then 255 - x on flipped samples.  normal_out [B][H][W][3] (the flip itself is applied by
 *   the readers below).
 * b200_data_resize_u8: Pillow's BILINEAR resize of uint8 [B][H][W][C] to [B][OH][OW][C]: the horizontal pass into
 *   tmp [B][H][OW][C], then the vertical pass.  Output o of an axis reads taps min[o] + j, j < ks, with 22-bit
 *   weights k[o * ks + j] (host-built tables on the device); flipped samples read mirrored source columns.
 * b200_data_depth_gather: dst [B][OH][OW] fp32 = src[b][rows[i]][cols[j]] (column W - 1 - cols[j] when flipped), from
 *   src_m (fp32 metres) or src_cm (uint16 centimetres, float32(cm) / 100.0) -- exactly one non-NULL.
 * b200_data_depth_range: per image, over the pixels near < d < far of depth [B][HW]: torch.quantile at 0.02 and 0.98
 *   (fp32 rank q * (n - 1), torch's fused CPU lerp) into range [B][2]; flag[B] = 0 (no valid pixel), 1 (min == max)
 *   or 2.
 * b200_data_finalise: per output pixel of load.py:248-281: rgb / normal read at (top + i, left + j) of [B][H][W][3]
 *   (mirrored, and 255 - x on the normal, when flipped); depth [B][OH][OW] from b200_data_depth_gather.  Writes
 *   rgb_out [B][3][OH][OW] = x / 255 * 2 - 1, the valid mask [B][OH][OW] (bytes), metric [B][OH][OW] (clamped, invalid
 *   pixels at max), depth_out [B][3][OH][OW] normalised to [-1, 1], normal_out [B][3][OH][OW] (F.normalize, zero where
 *   invalid); flag 0 / 1 give zero depth and metric, flag 1 also an empty mask. */
int b200_data_hypersim_source(const unsigned short* depth_mm, const unsigned char* normal, const unsigned char* flip,
                              int B, int H, int W, const double* inv_k, float* depth_m, unsigned char* normal_out,
                              void* stream);
int b200_data_resize_u8(const unsigned char* src, int B, int H, int W, int C, int OH, int OW, const int* xmin,
                        const int* xk, int xks, const int* ymin, const int* yk, int yks, const unsigned char* flip,
                        unsigned char* tmp, unsigned char* dst, void* stream);
int b200_data_depth_gather(const float* src_m, const unsigned short* src_cm, int B, int H, int W, int OH, int OW,
                           const int* rows, const int* cols, const unsigned char* flip, float* dst, void* stream);
int b200_data_depth_range(const float* depth, int B, long long HW, float near_plane, float far_plane, float* range,
                          int* flag, void* stream);
int b200_data_finalise(const unsigned char* rgb, const unsigned char* normal, int B, int H, int W, int top, int left,
                       const unsigned char* flip, const float* depth, int OH, int OW, float near_plane,
                       float far_plane, const float* range, const int* flag, float* rgb_out, float* depth_out,
                       float* metric_out, float* normal_out, unsigned char* mask_out, void* stream);

/* Virtual KITTI 2 training normals (ABI 16): D2NT "v3" of depth-to-normal-translator/python/gen_vkitti_normals.py
 * (DAG-filtered depth gradients, the depth-to-normal translation, the DLF-alpha MRF refinement) on uint16
 * centimetre depth [B][H][W], H, W >= 3, with intrinsics fx, fy, u0, v0 (float32, as the script's torch tensor holds
 * them).  out [B][H][W][3] uint16 = (-n + 1) * 32767.5 truncated, in the array order cv2.imwrite takes after the
 * script's cvtColor(RGB2BGR): z, y, x.  Bitwise the script's output with its fp32 np.power(e, -lap) replaced by the
 * correctly rounded fp32 value (DESIGN.md §3.11).  Nothing syncs the host. */
int b200_data_vkitti_normals(const unsigned short* depth_cm, int B, int H, int W, float fx, float fy, float u0,
                             float v0, unsigned short* out, void* stream);
/* The kernel's float32(e) ** -x (x >= 0, fp32 [n]) on its own, for testing the correct rounding: out[i] as
 * b200_data_vkitti_normals computes it; force_slow != 0 takes the double-double path for every element; slow_count
 * (device, nullable, not reset) is incremented once per element that took the double-double path. */
int b200_debug_pow_e32_neg(const float* x, long long n, int force_slow, float* out, unsigned int* slow_count,
                           void* stream);

/* Hypersim preprocessing (ABI 17): Marigold's script/dataset_preprocess/hypersim/preprocess_hypersim.py per frame,
 * for B frames of radiance rgb [B][H][W][3] and distance dist [B][H][W] (fp32, or fp16 where *_half != 0; both taken
 * exactly to fp64 as the script's astype(float)) and render_entity_id [B][H][W] int32.  bgr [B][H][W][3] uint8 = the
 * tone-mapped colour in the order cv2.imwrite takes after the script's cvtColor(RGB2BGR); depth_mm [B][H][W] uint16 =
 * the plane depth (distance / ||(x, y, focal)||_fp32 * focal) times 1000, 0 where entity id == -1, through NumPy's
 * wrapping float64 -> uint16 cast.  scale_num is the tone map's pow(0.8, 1 / (1 / 2.2)), computed on the host.
 * error_flag[b] (int32 [B], device) is set nonzero where frame b holds an entity id of 0, which the script asserts
 * against.  stats_out (device, nullable) receives [B][2] fp64 per frame: the 90th-percentile brightness (NaN when
 * the frame has no valid pixel) and the tone map's scale.  Bitwise the script's output with its np.power correctly
 * rounded (DESIGN.md §3.12).  workspace is device memory of at least b200_data_hypersim_workspace_bytes(B, H, W)
 * bytes, 8-byte aligned.  Nothing syncs the host. */
long long b200_data_hypersim_workspace_bytes(int B, int H, int W);
int b200_data_hypersim_frames(const void* rgb, int rgb_half, const void* dist, int dist_half, const int* entity_id,
                              int B, int H, int W, double focal, double scale_num, unsigned char* bgr,
                              unsigned short* depth_mm, int* error_flag, double* stats_out, void* workspace,
                              long long workspace_bytes, void* stream);
/* The tone map's power on its own, for testing the correct rounding: for m = x[i] (fp64 [n], the clamped scale * x),
 * p_out[i] = the pow(m, 1 / 2.2) b200_data_hypersim_frames uses (the correctly rounded value wherever it decides the
 * level) and level_out[i] = its uint8 level; force_slow != 0 takes the double-double path for every finite m > 0;
 * slow_count (device, nullable, not reset) is incremented once per element that took it. */
int b200_debug_hypersim_pow(const double* x, long long n, int force_slow, double* p_out, unsigned char* level_out,
                            unsigned int* slow_count, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200_E2EFT_H_ */
