/*
 * libudh.so — C ABI of the H100-native unsupervised-deep-homography hot path.
 *
 * The reference (tynguyen/unsupervisedDeepHomographyRAL2018) is a pure-Python TF1 graph and has no FFI of its
 * own; each entry point below replaces the group of TF ops cited next to it (file:line under /root/reference/code).
 * The Python mirror of the reference API (HomographyModel, transformer, the CLI) sits on top of this ABI and is
 * the binding a maintainer would use (INTEGRATION.md).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller unless the name says `host`; the library never
 *     allocates device memory — scratch is passed in as a workspace sized by the *_workspace_bytes query;
 *   - tensors are dense NHWC fp32 (the reference's layout and dtype); indices are int32;
 *   - every call is asynchronous on the `stream` argument (a cudaStream_t passed as void*) and re-entrant across
 *     streams; no exceptions cross the boundary: return 0 on success, a negative UDH_E* code otherwise and
 *     udh_last_error() gives the message (thread-local);
 *   - there is no CPU fallback: without a CUDA device every compute entry point returns UDH_ECUDA.
 */
#ifndef UDH_H_
#define UDH_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UDH_OK 0
#define UDH_EINVAL (-1) /* bad argument (shape, alignment, null pointer)   */
#define UDH_ECUDA (-2)  /* CUDA runtime / launch error                      */
#define UDH_ENOSUP (-3) /* configuration not supported by this build        */
#define UDH_EWS (-4)    /* workspace too small                              */

/* numeric mode of the regressor (udh_cnn_*).  FP32: CUDA-core fp32 everywhere — the parity mode.
 * BF16: wgmma bf16 tensor-core tiles with fp32 register accumulation, fp32 master weights — the throughput mode. */
#define UDH_NUMERIC_FP32 0
#define UDH_NUMERIC_BF16 1
/* BF16X3: the same wgmma tiles with ERROR-COMPENSATED operands: every fp32 activation / gradient / weight travels as two
 * 16-bit limbs (x = hi + lo) and every product is evaluated as lo.hi + hi.hi + hi.lo with fp32 register accumulation, so the
 * regressor reproduces fp32 arithmetic to ~1e-5 relative (the tensor-core parity mode; three MMA passes per product). */
#define UDH_NUMERIC_BF16X3 2

/* photometric loss selector for udh_warp_loss_bwd (reference --loss_type, homography_CNN_synthetic.py:51) */
#define UDH_LOSS_L1 0        /* homography_model.py:328 */
#define UDH_LOSS_REC 1       /* homography_model.py:303 */
#define UDH_LOSS_L1_SMOOTH 2 /* homography_model.py:136-139,340 */
#define UDH_LOSS_NCC 3       /* homography_model.py:161-166,351 */
#define UDH_LOSS_CUSTOM 4    /* per-pixel d loss / d pred supplied by the caller (ssim_loss: udh_ssim_bwd) */

/* slots of the `sums` accumulator (double[UDH_NSUMS]) filled by udh_warp_loss_fwd / udh_ssim_fwd */
#define UDH_SUM_ABS 0   /* sum |pred - I2|            */
#define UDH_SUM_SQ 1    /* sum (pred - I2)^2          */
#define UDH_SUM_HUBER 2 /* sum huber_1(pred - I2)     */
#define UDH_SUM_XY 3    /* sum pred * I2              */
#define UDH_SUM_XX 4    /* sum pred^2                 */
#define UDH_SUM_YY 5    /* sum I2^2                   */
#define UDH_SUM_SSIM 6  /* sum clip((1-SSIM)/2,0,1)   */
#define UDH_NSUMS 8

/* slots of the float[UDH_NLOSSES] written by udh_photo_losses_finalize (homography_model.py:291-296) */
#define UDH_L_REC 0
#define UDH_L_SSIM 1
#define UDH_L_L1 2
#define UDH_L_L1_SMOOTH 3
#define UDH_L_NCC 4
#define UDH_NLOSSES 8

/* slots of the float[UDH_NMETRICS] written by udh_h4p_loss (homography_model.py:274-281,288) */
#define UDH_M_H_LOSS 0         /* sqrt(mean_{B x 8} (pred-gt)^2)                       */
#define UDH_M_BOUNDED_H_LOSS 1 /* mean_b of per-sample RMSE, identity-bounded          */
#define UDH_M_NUM_FAIL 2       /* #samples with RMSE >= identity RMSE                  */
#define UDH_M_ACE 3            /* mean Euclidean corner distance (literature's metric) */
#define UDH_NMETRICS 4

int udh_version(void);
const char* udh_last_error(void);
/* 1 when a CUDA device is usable from this process, 0 otherwise (never throws). */
int udh_device_available(void);

/* ---- Row D: HomographyModel.solve_DLT (homography_model.py:169-250, utils/utils.py:11-122) ------------------
 * pts1[B,8] (x,y)x[TL,TR,BR,BL], h4p[B,8] -> H[B,9] row-major, h33 = 1, mapping pts1 -> pts1+h4p in pixels.
 * One warp per sample: 8x8 [A|b] in registers, LU with partial pivoting through warp shuffles
 * (replaces the 8 tf.matmul with Aux_M*, stack/transpose and tf.matrix_solve at :223-242). */
int udh_dlt_fwd(const float* pts1, const float* h4p, float* H, int B, void* stream);
/* TF autodiff of the above: dH[B,9] -> dh4p[B,8] (solve A^T lambda = dH[0:8]; dA = -lambda h^T, db = lambda). */
int udh_dlt_bwd(const float* pts1, const float* h4p, const float* H, const float* dH, float* dh4p, int B, void* stream);

/* ---- Row W+L: HomographyModel.transform + photometric losses ----------------------------------------------
 * (homography_model.py:252-269,291-296,328; utils/tf_spatial_transformer.py:76-247)
 * Fused: H' = M^-1 H M, homography warp of I[B,img_h,img_w,C] (C in {1,3}), channel mean, and ONLY the window
 * the reference gathers with patch_indices (a pw x ph rectangle whose first index patch_indices[b*idx_stride]
 * = y0*img_w + x0 gives its origin; patch_indices == NULL means origin (0,0)), compared with I2[B,ph,pw].
 * pred (nullable) receives pred_I2[B,ph,pw]; sums (double[UDH_NSUMS], caller-zeroed) accumulates the
 * reductions every photometric loss needs.  pw must be a multiple of 4. */
int udh_warp_loss_fwd(const float* I, int C, int img_h, int img_w, const float* H, const float* I2,
                      const int32_t* patch_indices, int64_t idx_stride, int pw, int ph, float* pred, double* sums,
                      int B, void* stream);
/* all_sums = 0: accumulate sums[UDH_SUM_ABS] only (what l1_loss needs) — the variant BASELINE configs[3] measures. */
int udh_warp_loss_fwd_ex(const float* I, int C, int img_h, int img_w, const float* H, const float* I2,
                         const int32_t* patch_indices, int64_t idx_stride, int pw, int ph, float* pred, double* sums,
                         int all_sums, int B, void* stream);
/* d loss / d H [B,9] for loss_type in UDH_LOSS_*; `sums` is the forward accumulator (needed by REC),
 * upstream multiplies the gradient (1.0 for a plain backward).  Recomputes the warp; no image-sized
 * intermediates.  scratch: float[B*9], caller-provided. */
int udh_warp_loss_bwd(const float* I, int C, int img_h, int img_w, const float* H, const float* I2,
                      const int32_t* patch_indices, int64_t idx_stride, int pw, int ph, int loss_type,
                      const double* sums, float upstream, float* dH, float* scratch, int B, void* stream);
/* same, with the per-pixel upstream gradient dpred[B,ph,pw] for UDH_LOSS_CUSTOM (NULL otherwise) */
int udh_warp_loss_bwd_ex(const float* I, int C, int img_h, int img_w, const float* H, const float* I2,
                         const int32_t* patch_indices, int64_t idx_stride, int pw, int ph, int loss_type,
                         const double* sums, const float* dpred, float upstream, float* dH, float* scratch, int B, void* stream);
/* d mean(clip((1-SSIM)/2,0,1)) / d pred -> dpred[B,ph,pw] (homography_model.py:141-158,316); feed to udh_warp_loss_bwd_ex. */
int udh_ssim_bwd(const float* pred, const float* I2, int pw, int ph, float* dpred, int B, void* stream);
/* SSIM diagnostic (homography_model.py:141-158): adds sum over the VALID 3x3 grid into sums[UDH_SUM_SSIM]. */
int udh_ssim_fwd(const float* pred, const float* I2, int pw, int ph, double* sums, int B, void* stream);
/* losses[UDH_NLOSSES] from sums; n = B*ph*pw, n_ssim = B*(ph-2)*(pw-2). */
int udh_photo_losses_finalize(const double* sums, double n, double n_ssim, float* losses, void* stream);

/* ---- the `transformer` operator (utils/tf_spatial_transformer.py:18,249-251) --------------------------------
 * U[B,H,W,C], theta[B,9] (normalised homography H'), -> out[B,out_h,out_w,C]; reference semantics including
 * the linspace grid, the t_s epsilon rule and clip-then-weight bilinear sampling. */
int udh_transformer_fwd(const float* U, const float* theta, float* out, int B, int H, int W, int C, int out_h,
                        int out_w, void* stream);

/* ---- Row L (h4p part): h_loss and the test-mode metrics (homography_model.py:274-281,288) -------------------
 * metrics: float[UDH_NMETRICS]; per_sample (nullable): float[B] batch_h_loss; dpred (nullable): d h_loss / d pred. */
int udh_h4p_loss(const float* pred, const float* gt, int B, float* metrics, float* per_sample, float* dpred,
                 void* stream);

/* ---- Row C: HomographyModel._vgg (homography_model.py:88-133) -----------------------------------------------
 * params / grads: the flat fp32 buffer laid out by udh_param_offset (TF-Slim checkpoint shapes: HWIO conv
 * kernels, [in,out] fc kernels, NHWC flatten).  I1, I2: [B,P,P] gray patches (the two channels of model_input,
 * homography_model.py:359, read in place — no concat copy).  train != 0 enables dropout(keep 0.5) after conv4_2
 * and fc1 with masks drawn from `seed` (kept in the workspace for the backward and readable with
 * udh_cnn_dropout_masks).  The workspace keeps the activations between fwd and bwd. */
size_t udh_cnn_workspace_bytes(int B, int P, int numeric_mode);
/* call once after allocating the workspace (zeroes the borders of the padded bf16 streams of UDH_NUMERIC_BF16). */
int udh_cnn_workspace_init(void* ws, size_t ws_bytes, int B, int P, int numeric_mode, void* stream);
int udh_cnn_fwd(const float* params, const float* I1, const float* I2, float* h4p, void* ws, size_t ws_bytes, int B,
                int P, int train, uint64_t seed, int numeric_mode, void* stream);
/* flags: UDH_FWD_FC1_MIRROR_CURRENT — the workspace's bf16 copy of fc1's weights already matches `params`
 * (udh_adam_step_mirror wrote it, or a previous forward did and params are unchanged): skip the conversion. */
#define UDH_FWD_FC1_MIRROR_CURRENT 1
int udh_cnn_fwd_ex(const float* params, const float* I1, const float* I2, float* h4p, void* ws, size_t ws_bytes, int B,
                   int P, int train, uint64_t seed, int numeric_mode, int flags, void* stream);
/* dh4p[B,8] -> grads (ACCUMULATED into the flat buffer: caller zeroes it once per step). */
int udh_cnn_bwd(const float* params, const float* I1, const float* I2, const float* dh4p, float* grads, void* ws,
                size_t ws_bytes, int B, int P, int train, int numeric_mode, void* stream);
/* The same backward in two halves, so the caller can start the allreduce of the fully connected gradients (98 % of the
 * bytes: fc1 is 33.5 M of the 34.2 M parameters) while the convolution backward is still running:
 * UDH_BWD_HEAD = fc2 + fc1 (leaves d(conv4_2 pre-activation) in the workspace), UDH_BWD_CONVS = the conv stack. */
#define UDH_BWD_ALL 0
#define UDH_BWD_HEAD 1
#define UDH_BWD_CONVS 2
int udh_cnn_bwd_phase(const float* params, const float* I1, const float* I2, const float* dh4p, float* grads, void* ws,
                      size_t ws_bytes, int B, int P, int train, int numeric_mode, int phase, void* stream);
/* device pointers (inside ws) of the uint8 keep-masks of the last train-mode forward: [B,(P/8)^2*128] and [B,1024]. */
int udh_cnn_dropout_masks(void* ws, size_t ws_bytes, int B, int P, int numeric_mode, const uint8_t** mask_conv4,
                          const uint8_t** mask_fc1);
/* device pointer (inside ws) of a saved activation, for tests: layer 0..7 = conv outputs, 8..10 = pool1..3,
 * 11 = fc1 (post-ReLU, pre-dropout).  *numel receives the element count. */
int udh_cnn_activation(void* ws, size_t ws_bytes, int B, int P, int numeric_mode, int layer, const float** ptr,
                       size_t* numel);
/* layout of the flat parameter buffer: tensor index 0..19 = (conv w, conv b) x 8, fc1 w, fc1 b, fc2 w, fc2 b. */
int udh_param_offset(int P, int tensor, size_t* offset_floats, size_t* numel);
size_t udh_param_total_floats(int P);

/* ---- Row O: TF-1 Adam (homography_CNN_synthetic.py:183,278) --------------------------------------------------
 * g' = g * grad_scale (1/world_size folds get_average_grads, utils/utils.py:380-403, into the update);
 * m = b1 m + (1-b1) g'; v = b2 v + (1-b2) g'^2; p -= alpha_t * m / (sqrt(v) + eps), alpha_t = lr_t*sqrt(1-b2^t)/(1-b1^t)
 * computed by the caller (t is 1-based).  If zero_grad != 0 the gradient buffer is cleared in the same pass. */
int udh_adam_step(float* p, float* g, float* m, float* v, size_t n, float alpha_t, float beta1, float beta2,
                  float eps, float grad_scale, int zero_grad, void* stream);
/* Same update, fused with the refresh of a bf16 weight mirror (UDH_NUMERIC_BF16): the updated parameters of the float
 * range [mirror_begin, mirror_begin + mirror_count) are also written, rounded to bf16, to `mirror`; with
 * mirror_keep_grad != 0 the gradient of that range is not cleared (its producer stores rather than accumulates).
 * udh_cnn_fc1_mirror names the range and the buffer for fc1's weights; a forward pass that follows may then be given
 * UDH_FWD_FC1_MIRROR_CURRENT and skips its own fp32 -> bf16 conversion of the 128 MB tensor. */
int udh_adam_step_mirror(float* p, float* g, float* m, float* v, size_t n, float alpha_t, float beta1, float beta2,
                         float eps, float grad_scale, int zero_grad, void* mirror, size_t mirror_begin, size_t mirror_count,
                         int mirror_keep_grad, void* stream);
/* mirror_limbs = 2 (UDH_NUMERIC_BF16X3): the mirror holds two 16-bit planes of mirror_count elements each, hi then lo,
 * with p = hi + lo; mirror_limbs = 1 is udh_adam_step_mirror. */
int udh_adam_step_mirror_ex(float* p, float* g, float* m, float* v, size_t n, float alpha_t, float beta1, float beta2,
                            float eps, float grad_scale, int zero_grad, void* mirror, size_t mirror_begin, size_t mirror_count,
                            int mirror_keep_grad, int mirror_limbs, void* stream);
/* bf16 copy of fc1's weights inside the workspace: *mirror (NULL in UDH_NUMERIC_FP32), its float range in the flat
 * parameter buffer, and whether fc1's weight gradient is stored (1) or accumulated (0) by the backward pass. */
int udh_cnn_fc1_mirror(void* ws, size_t ws_bytes, int B, int P, int numeric_mode, void** mirror, size_t* param_begin,
                       size_t* count, int* grad_is_stored);

/* ---- one call per step -------------------------------------------------------------------------------------------
 * The reference runs a step as ONE sess.run([apply_grad_opt, losses...]) (homography_CNN_synthetic.py:335-345).
 * udh_step_forward_backward enqueues regressor forward, h4p losses (:274-288), DLT (:169-250), fused warp + all
 * photometric diagnostics (:252-269,291-296) and the backward of the selected loss on `stream`; the caller then runs the
 * gradient allreduce (N > 1) and udh_adam_step.  Every output buffer is caller-owned and reused step after step. */
#define UDH_STEP_ALL 0      /* forward + full backward                                                         */
#define UDH_STEP_FWD_HEAD 1 /* forward + backward of the fully connected head (then allreduce fc grads ...)    */
#define UDH_STEP_CONVS 2    /* ... while this runs: backward of the conv stack                                 */
#define UDH_STEP_FWD_ONLY 3 /* evaluation: forward, losses, metrics                                            */
#define UDH_STEP_LOSS_H 0
#define UDH_STEP_LOSS_L1 1
#define UDH_STEP_LOSS_REC 2
#define UDH_STEP_LOSS_L1_SMOOTH 3
#define UDH_STEP_LOSS_NCC 4
#define UDH_STEP_LOSS_SSIM 5
typedef struct {
  int B, P, img_h, img_w, C;      /* batch, patch size, image size, channels of I_aug (1 or 3) */
  int numeric_mode, loss_type, train;
  uint64_t seed;                  /* dropout seed of this step */
  const float* params; float* grads; void* ws; size_t ws_bytes;
  const float *I1, *I2, *I_aug, *pts1, *gt;   /* gt may be NULL (no h_loss / metrics) */
  const int32_t* patch_indices; int64_t idx_stride;
  float *h4p, *H, *pred_I2;       /* [B,8], [B,9], [B,P,P] (pred_I2 may be NULL: then no SSIM) */
  float *dh4p, *dH, *scratch;     /* [B,8], [B,9], [B,9] */
  float* dpred_map;               /* [B,P,P] scratch, only for UDH_STEP_LOSS_SSIM */
  double* sums;                   /* [UDH_NSUMS] */
  float *photo_losses, *h4p_metrics, *per_sample;   /* [UDH_NLOSSES], [UDH_NMETRICS], [B] or NULL */
  int fwd_flags;                  /* UDH_FWD_* */
} udh_step_args;
int udh_step_forward_backward(const udh_step_args* args, int phase, void* stream);

/* ---- device-side input pipeline (dataloader.py:99-100,172-177,203-227; SURVEY 8f item 1) ------------------------
 * I, I_prime: uint8 [B,img_h,img_w,3] decoded images; pts1 [B,8].  Writes the post-dataloader tensors the step
 * consumes: I_aug fp32 [B,img_h,img_w,3] (normalised with I's statistics), gray patches I1, I2 fp32 [B,P,P] at
 * (x0,y0) = pts1[0:2], and patch_origin[B] = y0*img_w + x0 (the first patch index of each sample). */
int udh_prep_inputs_u8(const uint8_t* I, const uint8_t* I_prime, const float* pts1, float* I_aug, float* I1, float* I2,
                       int32_t* patch_origin, int B, int img_h, int img_w, int P, void* stream);

/* Same pipeline with the reference's photometric augmentation (dataloader.py:163-169,323-375) fused in, and a GRAY warp
 * source: aug (nullable) = [B,11] {on, gamma, brightness, colour R/G/B for I, then the same five for I'} — joint
 * augmentation (train) passes the same five numbers twice, disjoint (test) two draws; gamma acts on the raw 0..255 values.
 * Outputs: I_gray [B,img_h,img_w] = channel mean of the normalised (augmented) I — the warp's channel mean commutes with
 * its linear sampling, so the warp kernel can read this plane with C = 1 (a third of the bytes); I_aug3 (nullable) the
 * 3-channel tensor of the reference contract; I1_aug, I2_aug [B,P,P] the CNN input / L1 target; I1, I2 (nullable, together)
 * the un-augmented patches (summaries only in the reference); patch_origin [B] (nullable). */
int udh_prep_inputs_u8_ex(const uint8_t* I, const uint8_t* I_prime, const float* pts1, const float* aug, float* I_gray, float* I_aug3,
                          float* I1, float* I2, float* I1_aug, float* I2_aug, int32_t* patch_origin, int B, int img_h, int img_w,
                          int P, void* stream);
/* ---- on-device synthetic pairs (utils/gen_synthetic_data.py:40-68; MS-COCO is not available offline) ---------------
 * udh_synth_scene_u8: seeded multi-octave texture I [B,img_h,img_w,3] uint8, patch corners pts1 [B,8] with
 * x0 in [rho, W-rho-P], y0 in [rho, Hh-rho-P] (:42-50) and integer corner perturbations gt [B,8] in [-rho, rho] (:53).
 * udh_dlt_fwd(pts1, gt) then gives H_gt (:56) and udh_warp_image_u8 the second image I' = uint8(warp(I, H_gt)) (:63-64,
 * numpy_spatial_transformer.py:131-146). */
int udh_synth_scene_u8(uint8_t* I, float* pts1, float* gt, int B, int img_h, int img_w, int P, int rho, uint64_t seed, void* stream);
int udh_warp_image_u8(const uint8_t* U, const float* H, uint8_t* out, int B, int img_h, int img_w, void* stream);

/* ---- report image of the test harnesses (utils/utils.py:209-307, save_correspondences_img) -----------------------------
 * udh_draw_report_u8: out [B,img_h,2*img_w,3] = [left | right], left = denorm(I') and right = denorm(I) when prime_left,
 *   else the other way round (denorm as in udh_ecc_prep_u8, aug nullable), with cv2's drawing on it byte for byte:
 *   verts [B,20,2] int32 = the prediction polygon (right-image coordinates, drawn on the right image alone), kp2 and kp1
 *   (thick-3 closed polylines, colour (2,10,240)), and 4 match lines start -> end (LINE_AA, each end circled, r = 7).
 *   Any int32 vertex is accepted; nothing outside the canvas is touched.  workspace: udh_draw_report_workspace_bytes. */
size_t udh_draw_report_workspace_bytes(int B);
int udh_draw_report_u8(const uint8_t* I, const uint8_t* I_prime, const float* aug, int prime_left, const int32_t* verts, uint8_t* out,
                       void* ws, size_t ws_bytes, int B, int img_h, int img_w, void* stream);

/* ---- direct-method baseline: cv2.findTransformECC, MOTION_HOMOGRAPHY (utils/direct_homography.py:8-57) ----------------
 * as homography_conventional_synthetic.py:186-223 runs it on the test set, batched.  Images are uint8 planes
 * [B,img_h,img_w]; W [B,9] row-major fp32 maps template pixels into the input image (WARP_INVERSE_MAP).
 * udh_ecc_prep_u8: the two gray planes the reference hands to ECC from the decoded I, I' [B,img_h,img_w,3] and the
 *   augmentation table of udh_prep_inputs_u8_ex (nullable): augment + normalise (fp32), denorm_img (fp64), astype(uint8),
 *   cvtColor(RGB2GRAY) (utils/utils.py:406-413, homography_conventional_synthetic.py:190-191).
 * udh_ecc_homography: gray_I is the template, gray_I' the input image; W_init [B,9] (nullable = identity); runs up to
 *   max_iters iterations, stopping early when |rho - rho_last| < eps.  Writes W, rho [B] (the last correlation coefficient),
 *   iters [B] (iterations entered) and status [B]: UDH_ECC_* — where cv2 raises, the sample stops with W as it was before
 *   that iteration's update.  workspace: udh_ecc_workspace_bytes.
 * udh_ecc_h4p: pred_h4p [B,8] = perspectiveTransform(pts1, inv(W)) - pts1 (zeros when status != 0 or W is singular),
 *   then values >= rho_clamp become 2 rho_clamp and values <= -rho_clamp become -2 rho_clamp.  With gt (nullable):
 *   h_loss [B] = RMSE(pred, gt) and fail [B] = 1 (not found; scores as pred = 0) or 2 (identity < h_loss: h_loss becomes
 *   the identity RMSE), else 0 — the harness's rules, not udh_h4p_loss's. */
#define UDH_ECC_OK 0
#define UDH_ECC_NAN 1     /* rho is NaN ("NaN encountered.")                                     */
#define UDH_ECC_NOCONV 2  /* lambda_d <= 0 ("The algorithm stopped before its convergence ...") */
size_t udh_ecc_workspace_bytes(int B, int img_h, int img_w);
int udh_ecc_prep_u8(const uint8_t* I, const uint8_t* I_prime, const float* aug, uint8_t* gray_I, uint8_t* gray_I_prime, int B,
                    int img_h, int img_w, void* stream);
int udh_ecc_homography(const uint8_t* tmpl, const uint8_t* input, const float* W_init, int max_iters, double eps, float* W,
                       double* rho, int32_t* iters, int32_t* status, void* ws, size_t ws_bytes, int B, int img_h, int img_w,
                       void* stream);
/* udh_ecc_homography_split: udh_ecc_homography's contract (arguments, outputs, statuses, cv2 semantics) with each pair's
 *   pixel sums split over many CTAs, for a few large pairs.  The tiling depends on img_h x img_w only: a pair's result is
 *   bit-identical alone or in any batch.  Sums are added in a fixed order (no atomics); the call enqueues max_iters
 *   iterations of three launches each and returns without synchronising.  workspace: udh_ecc_split_workspace_bytes. */
size_t udh_ecc_split_workspace_bytes(int B, int img_h, int img_w);
int udh_ecc_homography_split(const uint8_t* tmpl, const uint8_t* input, const float* W_init, int max_iters, double eps, float* W,
                             double* rho, int32_t* iters, int32_t* status, void* ws, size_t ws_bytes, int B, int img_h, int img_w,
                             void* stream);
/* udh_debug_ecc_layout: where the ECC workspaces keep their intermediates, for tests that read them (byte offsets).
 *   off[0]: the blurred fp32 planes [2][B][img_h][img_w], template planes then input planes — the whole of
 *     udh_ecc_homography's workspace, and the first part of udh_ecc_homography_split's;
 *   split kernel only: off[1] the per-pair states, off[2] slab1 fp64 [B][tiles][5] (per tile: mask count n, sum Iw,
 *     sum Iw^2, sum T, sum T^2), off[3] slab2 fp64 [B][tiles][53] (per tile: the Hessian's upper triangle row by row,
 *     the 8 image projections, the 8 template projections, the correlation).  *tiles = the tiles of 16384 row-major
 *     pixels.  After the call the slabs hold the last iteration's sums (with max_iters = 1: the first one's). */
int udh_debug_ecc_layout(int B, int img_h, int img_w, size_t off[4], int* tiles);
int udh_ecc_h4p(const float* W, const int32_t* status, const float* pts1, const float* gt, float rho_clamp, float* pred_h4p,
                float* h_loss, int32_t* fail, int B, void* stream);
/* udh_ecc_corr_h4p: the real-data harness's metric (homography_conventional_real.py:213-246, return_h_inv = False).
 *   gt [B,16] fp32: four correspondences clicked on 480x640 frames; corr1 = gt[0:8] / 2, corr2 = gt[8:16] / 2.
 *   status == 0: pred_h4p [B,8] = perspectiveTransform(corr1, W) - corr1 (W NOT inverted), clamped to +-80;
 *     h_loss [B] = RMSE(pred + corr1, corr2) in fp32; fail = 2 and h_loss = the identity RMSE when that is smaller.
 *   status != 0: pred_h4p = 0, fail = 1, h_loss = the identity RMSE computed in float64 (no identity bound). */
int udh_ecc_corr_h4p(const float* W, const int32_t* status, const float* gt, float* pred_h4p, double* h_loss, int32_t* fail, int B,
                     void* stream);

/* ---- real-data input pipeline (dataloader.py:146-200), bit-identical to the host's cv2 / NumPy arithmetic ----------------
 * udh_resize_area_up_u8: cv2.resize(src, (dst_w, dst_h), INTER_AREA) on n uint8 [src_h,src_w,3] images, dst larger on both
 *   axes.  tab (device, int32): xsrc[dst_w], xa0[dst_w], xa1[dst_w], ysrc[dst_h], ya0[dst_h], ya1[dst_h] — first source
 *   index and the two 11-bit coefficients per output column / row, as OpenCV computes them (ops.linear_area_table).
 * udh_real_prep: full-size uint8 I, I' [B,full_h,full_w,3] -> the loader's four network-size fp32 images [B,img_h,img_w,3]:
 *   I_plain = T0[I], I_prime_plain = T1[I'], I_aug = T2[I], I_prime_aug = T3[I'], each AREA-downscaled when the sizes
 *   differ.  luts (device) [B][4][256][3] fp32 are the per-value tables T0..T3 (augment + normalise).  tab (device, int32,
 *   nullable when the sizes are equal): nx, ny, xofs[img_w+1], xsrc[nx], xw[nx], yofs[img_h+1], ysrc[ny], yw[ny] (weights
 *   as fp32 bits): OpenCV's computeResizeAreaTab entries of each output column / row in table order (ops.area_table);
 *   max_rows = the most entries of one output row.  The downscale is resizeArea's generic path: sequential fp32 sums, no FMA.
 *   Any full size: an output row's source rows are staged in shared memory (udh_real_prep_smem_bytes(max_rows, full_w))
 *   when that fits in 227 KB, and read from global memory otherwise, with the same sums in the same order. */
int udh_resize_area_up_u8(const uint8_t* src, const int32_t* tab, uint8_t* dst, int n, int src_h, int src_w, int dst_h, int dst_w,
                          void* stream);
/* udh_resize_linear_u8: cv2.resize(src, (dst_w, dst_h)) with the default INTER_LINEAR on n uint8 [src_h,src_w,3] images, any
 *   sizes (down or up).  The kernel of udh_resize_area_up_u8 with OpenCV's INTER_LINEAR table (ops.linear_table):
 *   f = (float)((d + 0.5) * scale - 0.5), floor, coefficients in float rounded to 11 bits; tab = xsrc[dst_w], xa0, xa1,
 *   ysrc[dst_h], ya0, ya1, ysrc1[dst_h]: columns clamp index and coefficient at the borders, rows keep the coefficients
 *   and give both (clamped) source rows. */
int udh_resize_linear_u8(const uint8_t* src, const int32_t* tab, uint8_t* dst, int n, int src_h, int src_w, int dst_h, int dst_w,
                         void* stream);
size_t udh_real_prep_smem_bytes(int max_rows, int full_w);
int udh_real_prep(const uint8_t* I, const uint8_t* I_prime, const float* luts, const int32_t* tab, int max_rows, int B, int full_h,
                  int full_w, int img_h, int img_w, float* I_plain, float* I_prime_plain, float* I_aug, float* I_prime_aug, void* stream);

/* ---- baseline-JPEG decode, bit-identical to cv2.imread(..., IMREAD_COLOR) + BGR->RGB (libjpeg-turbo defaults) --------
 * Accepted: baseline Huffman 8-bit (SOF0, SOF1), one interleaved scan, gray or YCbCr with luma sampling 1x1, 2x1 or 2x2 and
 * chroma 1x1; any size; restart intervals; APPn / COM skipped.  Everything else is rejected with a UDH_JPEG_R_* reason.
 * udh_jpeg_parse (host): one file -> info; returns UDH_OK with info->reason set, or UDH_EINVAL on a null pointer.
 * udh_jpeg_plan_bytes / udh_jpeg_plan (host): N files, concatenated in `data` with file k at [offsets[k], offsets[k+1]),
 *   all h x w and supported -> the packed descriptor (tables + restart segments).  plan_bytes returns 0 when the plan
 *   cannot be built; udh_jpeg_plan then returns UDH_ENOSUP (a file is not supported) or UDH_EINVAL (wrong size).
 * udh_jpeg_decode (device): plan_host is the plan as udh_jpeg_plan wrote it, plan_dev a 16-byte aligned device copy,
 *   data the same concatenated bytes on the device; writes out [N,h,w,3] uint8 RGB and status [N] (0, or a
 *   UDH_JPEG_E_* code: that image's output is undefined, the other images are unaffected).
 *   workspace: udh_jpeg_plan_workspace_bytes(plan_host), 16-byte aligned.  It equals udh_jpeg_workspace_bytes(N, h, w)
 *   unless the plan has a long segment (128 kB or more of entropy-coded data: a camera frame without restart markers);
 *   those are decoded by the parallel path, many threads per segment, with the same output and status codes. */
#define UDH_JPEG_R_OK 0
#define UDH_JPEG_R_NOT_JPEG 1      /* no SOI marker (PNG, ...)                                         */
#define UDH_JPEG_R_TRUNCATED 2     /* malformed or truncated header                                     */
#define UDH_JPEG_R_NOT_BASELINE 3  /* progressive, lossless, hierarchical or arithmetic-coded           */
#define UDH_JPEG_R_PRECISION 4     /* not 8-bit samples                                                 */
#define UDH_JPEG_R_COMPONENTS 5    /* 2 or 4 components                                                 */
#define UDH_JPEG_R_RGB 6           /* RGB-coded (Adobe transform 0, or component ids 'R','G','B')       */
#define UDH_JPEG_R_SAMPLING_H 7    /* horizontal sampling other than 4:4:4 / 4:2:x (e.g. 4:1:1)         */
#define UDH_JPEG_R_SAMPLING_V 8    /* vertical-only chroma subsampling (e.g. 4:4:0)                     */
#define UDH_JPEG_R_ORIENTATION 9   /* EXIF orientation other than 1 (cv2.imread rotates the image)      */
#define UDH_JPEG_R_MULTI_SCAN 10   /* components spread over several scans                              */
#define UDH_JPEG_E_TRUNCATED 1     /* entropy-coded data ran out                                        */
#define UDH_JPEG_E_HUFFMAN 2       /* invalid Huffman code                                              */
#define UDH_JPEG_E_COEF 3          /* coefficient index past 63                                         */
typedef struct udh_jpeg_info {
  int32_t width, height, components;
  int32_t h_samp[3], v_samp[3];
  int32_t restart_interval; /* MCUs per restart interval, 0 = none */
  int32_t reason;           /* UDH_JPEG_R_*                         */
} udh_jpeg_info;
int udh_jpeg_parse(const uint8_t* data, int64_t nbytes, udh_jpeg_info* info);
size_t udh_jpeg_plan_bytes(const uint8_t* data, const int64_t* offsets, int n, int h, int w);
int udh_jpeg_plan(const uint8_t* data, const int64_t* offsets, int n, int h, int w, void* plan, size_t plan_bytes);
size_t udh_jpeg_workspace_bytes(int n, int h, int w);
int udh_jpeg_decode(const void* plan_host, const void* plan_dev, const uint8_t* data, uint8_t* out, int32_t* status, void* ws,
                    size_t ws_bytes, void* stream);
/* Lanes per image in the entropy-decode kernel (32: one warp per image, the default; 1: eight images share a warp).  For
 * the timing tool's comparison; process-wide. */
int udh_debug_jpeg_set_lanes(int lanes);
size_t udh_jpeg_plan_workspace_bytes(const void* plan_host);
/* Which segments plans made from now on send to the parallel entropy path (-1: those of 128 kB or more, the default;
 * 0: none; 1: all), and how many synchronisation rounds a segment gets before it falls back to the serial path
 * (0..16, default 16).  udh_debug_jpeg_parallel_segments: after udh_jpeg_decode (synchronises), how many of the plan's
 * segments the parallel path decoded (the others went to the serial path).  For tests and the timing tool; process-wide. */
int udh_debug_jpeg_set_parallel(int mode);
int udh_debug_jpeg_set_sync_rounds(int rounds);
int udh_debug_jpeg_parallel_segments(const void* plan_host, const void* ws, int32_t* count);

/* ---- baseline-JPEG encode, byte-identical to cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, quality]) ------------------
 * libjpeg-turbo's defaults: JFIF APP0, standard Huffman tables, ISLOW DCT, no restart markers; channels = 3 takes uint8 BGR
 * [n,h,w,3] and writes YCbCr 4:2:0, channels = 1 takes gray [n,h,w] and writes one component.  quality 1..100.
 * udh_jpeg_encode_capacity: the largest file an h x w image can encode to (every coefficient at its longest code, every
 *   byte stuffed), 0 on bad dimensions; size each output row with it, no dry run needed.
 * udh_jpeg_encode_workspace_bytes: device workspace of one call, 0 on bad dimensions.
 * udh_jpeg_encode (device): img [n,h,w,channels] uint8; out [n][cap] with cap >= the capacity; nbytes [n] int64 = the file
 *   length of each image (its bytes are out[k][0, nbytes[k])); status [n] int32 = 0, or nonzero when that image could not
 *   be encoded (its output is then undefined, the other images are unaffected).  n <= 65535 per call.  The library
 *   allocates nothing. */
int64_t udh_jpeg_encode_capacity(int h, int w, int channels);
size_t udh_jpeg_encode_workspace_bytes(int n, int h, int w, int channels);
int udh_jpeg_encode(const uint8_t* img, int n, int h, int w, int channels, int quality, uint8_t* out, int64_t cap, int64_t* nbytes,
                    int32_t* status, void* ws, size_t ws_bytes, void* stream);

/* ---- PNG decode, bit-identical to cv2.imread(..., IMREAD_COLOR) ------------------------------------------------------------
 * Accepted: non-interlaced, bit depth 8, colour type 0 (gray: replicated to 3 channels), 2 (RGB) or 6 (RGBA: alpha dropped),
 * every chunk's CRC correct, IEND present.  Ancillary chunks that do not change what cv2 returns are skipped: tEXt, zTXt,
 * iTXt, tIME and pHYs.  Any other chunk (gAMA, sBIT, tRNS, cHRM, sRGB, iCCP, eXIf, PLTE, APNG frames, ...) is rejected
 * with UDH_PNG_R_CHUNK, and everything else out of scope with its own UDH_PNG_R_* reason.
 * udh_png_parse (host): one file -> info; returns UDH_OK with info->reason set, or UDH_EINVAL on a null pointer.
 * udh_png_plan_bytes / udh_png_plan (host): N files, concatenated in `data` with file k at [offsets[k], offsets[k+1]), all
 *   h x w and supported -> the descriptor (plan) and the files' IDAT payloads, concatenated per file into `idat`
 *   (*idat_bytes of them; file k's zlib stream is contiguous).  plan_bytes returns 0 when the plan cannot be built;
 *   udh_png_plan then returns UDH_ENOSUP (a file is not supported) or UDH_EINVAL (wrong size).
 * udh_png_decode (device): plan_host as udh_png_plan wrote it, plan_dev a 16-byte aligned device copy, idat the payloads on
 *   the device; writes out [N,h,w,3] uint8 (BGR as cv2 returns it; RGB when rgb != 0) and status [N] (0, or a
 *   UDH_PNG_E_* code: that image's output is undefined, the other images are unaffected).  Workspace:
 *   udh_png_workspace_bytes(plan_host) (the filtered scanlines), 16-byte aligned. */
#define UDH_PNG_R_OK 0
#define UDH_PNG_R_NOT_PNG 1         /* no PNG signature                                               */
#define UDH_PNG_R_JPEG 2            /* a JPEG file (SOI marker)                                       */
#define UDH_PNG_R_TRUNCATED 3       /* a chunk other than IDAT runs past the end of the file         */
#define UDH_PNG_R_IDAT_TRUNCATED 4  /* an IDAT chunk runs past the end of the file                    */
#define UDH_PNG_R_CRC 5             /* a chunk's CRC does not match                                   */
#define UDH_PNG_R_NO_IEND 6         /* the chunks end without IEND                                    */
#define UDH_PNG_R_MALFORMED 7       /* no or invalid IHDR, IDAT chunks not consecutive, no IDAT       */
#define UDH_PNG_R_PALETTE 8         /* colour type 3                                                  */
#define UDH_PNG_R_DEPTH16 9         /* bit depth 16                                                   */
#define UDH_PNG_R_DEPTH_SUB8 10     /* bit depth 1, 2 or 4                                            */
#define UDH_PNG_R_INTERLACED 11     /* Adam7                                                          */
#define UDH_PNG_R_GRAY_ALPHA 12     /* colour type 4                                                  */
#define UDH_PNG_R_CHUNK 13          /* a chunk that may change what cv2 returns (see above)           */
#define UDH_PNG_E_TRUNCATED 1       /* the zlib stream ran out                                        */
#define UDH_PNG_E_ZLIB 2            /* bad zlib header (method, window, check bits, preset dictionary) */
#define UDH_PNG_E_BLOCK 3           /* bad block: type 3, stored length check, invalid code lengths   */
#define UDH_PNG_E_CODE 4            /* invalid literal/length or distance code                        */
#define UDH_PNG_E_DISTANCE 5        /* a distance beyond the output or the window                     */
#define UDH_PNG_E_ADLER 6           /* Adler-32 mismatch                                              */
#define UDH_PNG_E_SHORT 7           /* fewer bytes than h * (1 + w * channels)                        */
#define UDH_PNG_E_LONG 8            /* more bytes than h * (1 + w * channels)                         */
#define UDH_PNG_E_FILTER 9          /* a row's filter type above 4                                    */
typedef struct udh_png_info {
  int32_t width, height, bit_depth, color_type, interlace;
  int32_t channels;         /* samples per pixel in the file (1, 2, 3 or 4; 1 for a palette)    */
  int64_t idat_bytes;       /* the zlib stream's length (all IDAT payloads)                      */
  int32_t reason;           /* UDH_PNG_R_*                                                        */
  int32_t pad;
} udh_png_info;
int udh_png_parse(const uint8_t* data, int64_t nbytes, udh_png_info* info);
size_t udh_png_plan_bytes(const uint8_t* data, const int64_t* offsets, int n, int h, int w, int64_t* idat_bytes);
int udh_png_plan(const uint8_t* data, const int64_t* offsets, int n, int h, int w, void* plan, size_t plan_bytes, uint8_t* idat,
                 int64_t idat_bytes);
size_t udh_png_workspace_bytes(const void* plan_host);
int udh_png_decode(const void* plan_host, const void* plan_dev, const uint8_t* idat, uint8_t* out, int32_t* status, int rgb,
                   void* ws, size_t ws_bytes, void* stream);

/* ---- the dataset generator's warp (gen_synthetic_data.py:63-64), bit-identical to the reference's NumPy ------------------
 * udh_gen_warp_u8: bgr [n,h,w,3] uint8 (cv2's channel order), theta [n,9] float64 (row-major inv(M) inv(H_inverse) M on the
 *   [-1,1] grid) -> gray [n,h,w] = cv2.cvtColor(bgr, COLOR_RGB2GRAY), warped [n,h,w,3] = numpy_transformer(bgr, H_inverse)
 *   per channel, warped_gray [n,h,w] = numpy_transformer(gray, H_inverse): float64 throughout, astype(uint8) on the result.
 *   n <= 65535. */
int udh_gen_warp_u8(const uint8_t* bgr, const double* theta, int n, int h, int w, uint8_t* gray, uint8_t* warped,
                    uint8_t* warped_gray, void* stream);
/* udh_gray_u8: bgr [npx,3] uint8 -> gray [npx] with udh_gen_warp_u8's gray rule (cv2.cvtColor(bgr, COLOR_RGB2GRAY)). */
int udh_gray_u8(const uint8_t* bgr, int64_t npx, uint8_t* gray, void* stream);

/* ---- image alignment's warp -----------------------------------------------------------------------------------------
 * udh_warp_perspective_u8: cv2.warpPerspective(src, M, (dst_w, dst_h)) with its defaults (INTER_LINEAR, BORDER_CONSTANT,
 *   border value 0), bit for bit: src [n,h,w,c] uint8 (c = 1 or 3), M [n,9] float64 row-major (device), dst [n,dst_h,dst_w,c].
 *   M is inverted in float64 by cv2's 3x3 cofactor rule; source positions are rounded to 1/32 pixel in float64 (a zero
 *   denominator lands on source pixel (0, 0), as in cv2); 15-bit bilinear weights; taps outside the source read 0.
 *   n <= 65535, all sides < 32767.  oracle/warp_perspective.py restates it. */
int udh_warp_perspective_u8(const uint8_t* src, const double* M, uint8_t* dst, int n, int h, int w, int c, int dst_h, int dst_w,
                            void* stream);

/* ---- sequence mosaic ---------------------------------------------------------------------------------------------------
 * udh_mosaic_blend_u8: n frames warped onto one dst_h x dst_w canvas and blended with feathered integer weights
 *   (oracle/mosaic.py restates the rule).  Per canvas pixel and frame k, (X, Y) is the source position in 1/32 pixel that
 *   udh_warp_perspective_u8(frame k, M_k, dst_h, dst_w) computes, W its denominator before 32 / W; the pixel is valid for k
 *   iff W != 0, 0 <= X <= 32 (w_k - 1) and 0 <= Y <= 32 (h_k - 1).  v_k is that warp's output value and
 *   wt_k = 1 + min(min(X, 32 (w_k - 1) - X, Y, 32 (h_k - 1) - Y), 32 feather).  Per channel S = sum wt_k v_k, D = sum wt_k
 *   over the valid frames (64-bit integers); dst = (S + (D >> 1)) / D and mask = 255, or 0 and 0 where D = 0.
 *   frames [n] (host array of device pointers), frame k uint8 [h_k,w_k,c] (c = 1 or 3); sizes [n,2] int32 (host, h_k w_k);
 *   M [n,9] float64 row-major (device), frame k -> canvas; dst [dst_h,dst_w,c], mask [dst_h,dst_w] uint8 (device).
 *   tile_ptr [ntiles + 1] and tile_frames [tile_ptr[ntiles]] int32 (device, CSR): the frames whose footprint can reach each
 *   UDH_MOSAIC_TILE_H x UDH_MOSAIC_TILE_W canvas tile, tiles row-major, ceil(dst_w / UDH_MOSAIC_TILE_W) per row.  The lists
 *   must be conservative (a frame valid at a pixel is listed for its tile); a frame listed twice counts twice.
 *   Optional inputs (each may be null; gains and maps exclude each other):
 *   gains [n][3] float64 (device): v_k is compensated before it is weighted (exposure compensation's apply, below, with
 *     g = gains[k][c], channel 0's gain when c = 1).
 *   maps [n] (host): v_k is compensated by frame k's gain map (block exposure compensation's apply, below) at
 *     (x - x_lo, y - y_lo) of its rectangle rois[k], clamped to it.
 *   masks [n] (host array of device pointers): frame k counts only where its uint8 blend mask on the rectangle rois[k] is set.
 *   rois [n,4] int32 (host) x_lo, y_lo, x_hi, y_hi (exclusive), required with masks or maps: an empty rectangle keeps the
 *     frame out (its mask and map may then be null); a non-empty one lies inside the canvas and needs a non-null mask (with
 *     masks) and a well-formed map (with maps).
 *   ws: udh_mosaic_workspace_bytes(n) bytes of device memory (whichever inputs are given).  n <= 65535, all sides < 32767,
 *   0 <= feather <= 1024. */
#define UDH_MOSAIC_TILE_H 16
#define UDH_MOSAIC_TILE_W 64
typedef struct udh_map_tap {
  int32_t s0, s1; /* the two source columns (rows) of the map */
  float a0, a1;   /* their weights */
} udh_map_tap;
typedef struct udh_gain_map {
  const float* map;        /* device: bpy x bpx x channels float32 */
  const udh_map_tap* cols; /* device: one per ROI column */
  const udh_map_tap* rows; /* device: one per ROI row */
  int32_t bpx, bpy, channels, pad;
} udh_gain_map;
size_t udh_mosaic_workspace_bytes(int n);
int udh_mosaic_blend_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const double* gains, const udh_gain_map* maps,
                        const uint8_t* const* masks, const int32_t* rois, int n, int c, const int32_t* tile_ptr, const int32_t* tile_frames,
                        int dst_h, int dst_w, int feather, uint8_t* dst, uint8_t* mask, void* ws, size_t ws_bytes, void* stream);
/* udh_mosaic_multiband_u8: n frames blended onto one dst_h x dst_w canvas across frequency bands, byte for byte
 *   cv2.detail_MultiBandBlender(0, bands, CV_16S) on the CPU (oracle/multiband.py restates the rule).  Frame k is fed as
 *   udh_warp_perspective_u8(frame k, M_k, roi_h, roi_w) at the ROI's top-left (x_lo, y_lo), with mask 255 where that warp is
 *   valid (udh_mosaic_blend_u8's rule: W != 0 and the source position inside the frame) and 0 elsewhere.  Then, with
 *   B' = min(bands, ceil(log2(max(dst_h, dst_w)))) and the canvas padded to multiples of 2^B': each frame's rectangle is its
 *   ROI grown by 3 2^B' per side and aligned as cv2 does; the image is bordered BORDER_REFLECT, the weight (256 where the
 *   mask is set) a constant 0; G_{i+1} = pyrDown(G_i) in uint8 and W_{i+1} = pyrDown(W_i) in int16; L_i = G_i - pyrUp(G_{i+1})
 *   (L_B' = G_B'); per level acc += (int16)((L W) >> 8), wacc += W with wrapping int16 adds.  The blend normalises each level
 *   to (int16)((acc << 8) / (wacc + 1)) (0 where wacc = -1, where cv2 divides by zero), collapses from the top with
 *   pyrUp and saturating int16 adds, and crops; dst = saturate_u8 of that and mask = 255 where wacc_0 > 0, else both 0.
 *   frames [n] (host array of device pointers), frame k uint8 [h_k,w_k,3]; sizes [n,2] int32 (host); M [n,9] float64
 *   (device) frame k -> its ROI (M_canvas translated by (-x_lo, -y_lo)); rois [n,4] int32 (host) x_lo, y_lo, x_hi, y_hi
 *   (exclusive), non-empty and inside the canvas; dst [dst_h,dst_w,3] and mask [dst_h,dst_w] uint8 (device).  The sums are
 *   gathered per canvas pixel in int32 and stored once, so the bytes do not depend on the frames' order.  Only c = 3 (the
 *   blender takes 3 channels).  n <= 65535, sides < 32767, 0 <= bands <= 10.
 *   Optional inputs (each may be null; gains and maps exclude each other), applied to every pixel of the ROI warp, valid or
 *   not, before it is fed, as cv2's stitcher applies its compensator before the blender:
 *   gains [n][3] float64 (device): exposure compensation's apply with g = gains[k][c].
 *   maps [n] (host): block exposure compensation's apply with frame k's gain map at the ROI pixel; well-formed.
 *   masks [n] (host array of device pointers, each non-null): frame k's roi_h x roi_w blend mask, fed in place of its
 *     validity mask.
 *   ws: udh_mosaic_multiband_workspace_bytes(rois, n, dst_h, dst_w, bands) bytes of device memory (0: bad arguments). */
size_t udh_mosaic_multiband_workspace_bytes(const int32_t* rois, int n, int dst_h, int dst_w, int bands);
int udh_mosaic_multiband_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const double* gains,
                            const udh_gain_map* maps, const uint8_t* const* masks, const int32_t* rois, int n, int c, int dst_h, int dst_w,
                            int bands, uint8_t* dst, uint8_t* mask, void* ws, size_t ws_bytes, void* stream);
/* udh_debug_multiband_layout: where udh_mosaic_multiband_u8's workspace keeps the canvas pyramid, for tests that read it.
 *   off[i] (i <= B'): byte offset of level i, int16 [Hp >> i][Wp >> i][4] (acc's three channels, then wacc), as the feeds
 *   left it (the blend does not overwrite it); dims = {B', Hp, Wp}, the padded canvas. */
int udh_debug_multiband_layout(const int32_t* rois, int n, int dst_h, int dst_w, int bands, size_t off[11], int dims[3]);

/* ---- exposure compensation (cv2.detail_GainCompensator / ChannelsCompensator; oracle/exposure.py restates the rule) ----
 * apply: v' = saturate_u8(rint(v g)) in float64, ties to even, per channel (cv2.multiply(uint8, double)).
 * udh_mosaic_exposure_stats_u8: the compensators' per-pair statistics of the frames' ROI warps (udh_mosaic_multiband_u8's
 *   frames, M (frame -> ROI, device) and rois (host)), in one pass over the canvas.  For each listed pair p = (i, j), i <= j,
 *   over the canvas pixels where both ROI warps are valid, stats[p] (uint64, device) holds UDH_EXPOSURE_STATS sums: [0] the
 *   count; [1..3] frame i's channel sums; [4..6] frame j's; with norms, [7..9] and [10..12] frame i's and j's sums of
 *   q = sqrt(double(r^2 + g^2 + b^2)) 2^52 (an integer below 2^61) as three 21-bit limbs, sum q = [7] + [8] 2^21 + [9] 2^42:
 *   exact, rounded to double by the caller (without norms those six are 0).  Before the sums, frame k's values are
 *   compensated by history[0][k][c], then history[1][k][c], ... up to history[feeds - 1] ([feeds][n][3] float64, device):
 *   the images cv2's feed number `feeds` sees.  pair_ptr [n + 1] and pair_j [npairs] int32 (device): the CSR list of pairs
 *   (row i, ascending j >= i); list every pair whose ROIs intersect, the diagonal included.  Integer sums: the result does
 *   not depend on the frames' order or the run.  n <= UDH_EXPOSURE_MAX_FRAMES, feeds <= UDH_EXPOSURE_MAX_FEEDS, canvas
 *   sides < 32767 (so a pair's count stays below 2^31).  ws: udh_mosaic_exposure_workspace_bytes(n) bytes of device memory. */
#define UDH_EXPOSURE_MAX_FRAMES 1024
#define UDH_EXPOSURE_MAX_FEEDS 16
#define UDH_EXPOSURE_STATS 13
size_t udh_mosaic_exposure_workspace_bytes(int n);
int udh_mosaic_exposure_stats_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const int32_t* rois, int n,
                                 const int32_t* pair_ptr, const int32_t* pair_j, int npairs, const double* history, int feeds,
                                 int norms, int dst_h, int dst_w, uint64_t* stats, void* ws, size_t ws_bytes, void* stream);

/* ---- block exposure compensation (cv2.detail_BlocksGainCompensator / BlocksChannelsCompensator; oracle/exposure_blocks.py)
 * Each fed frame's ROI (roi_w x roi_h) is cut into bpx x bpy blocks of bw x bh pixels (bpx = ceil(roi_w / block),
 * bw = ceil(roi_w / bpx), likewise in y); blocks are numbered frame-major, then row-major, frame k's from boff[k].
 * udh_mosaic_exposure_block_stats_u8: udh_mosaic_exposure_stats_u8's statistics per block pair.  For each listed frame pair
 *   p = (i, j), i <= j, over the ROIs' intersection the block columns of both frames merge: a pixel in block column bx_i of
 *   frame i and bx_j of frame j lies in cell column (bx_i - bx_i0) + (bx_j - bx_j0) (bx_i0, bx_j0: the columns at the
 *   intersection's left edge), likewise in y, and cell (cx, cy) is slot cell_off[p] + cy cell_nx[p] + cx of stats
 *   (uint64 [slots][UDH_EXPOSURE_STATS], device, zeroed here): the same 13 sums over the pixels of that block pair where
 *   both ROI warps are valid.  A frame's pair with itself gives each block's own count at cell (2 bx, 2 by).  blocks
 *   (host int32 [n][4]): bw, bh, bpx, bpy per frame; boff (host int64 [n]).  history [feeds][nblocks][3] float64 (device): a
 *   pixel of block b is compensated by history[0][b][c], then history[1][b][c], ... (cv2's feeds over the blocks).
 *   cell_off int64 [npairs], cell_nx int32 [npairs] (device).  Limits as udh_mosaic_exposure_stats_u8, nblocks <=
 *   UDH_EXPOSURE_MAX_BLOCKS.  ws: udh_mosaic_exposure_block_workspace_bytes(n).
 * udh_exposure_block_solve: x = A^-1 b for a symmetric positive definite A in CSR (row_ptr [n + 1] int32, col int32, val
 *   float64, device) by Jacobi-preconditioned conjugate gradients in float64, from x = 1, in one CTA whose reductions
 *   have a fixed order (the result does not depend on the run).  Stops when |r| <= tol |b| or after max_iter iterations;
 *   info (device int64 [2]) receives the iterations and the final |r| / |b| as a double's bits.  ws:
 *   udh_exposure_block_solve_workspace_bytes(n).
 * udh_exposure_gain_maps: per frame k its bpy x bpx map float32(gains[b][c]) (c < channels; gains [nblocks][3] float64,
 *   device), filtered twice by cv2.sepFilter2D([1/4, 1/2, 1/4] both ways, BORDER_REFLECT_101, float32: each output
 *   (a + c) 1/4 + b 1/2, the row pass then the column pass) into maps (float32 [nblocks][channels], device, frame k's at
 *   boff[k] channels).  blocks, boff as above (host).  ws: udh_exposure_gain_maps_workspace_bytes(nblocks, channels).
 * apply (the blends' maps): v at ROI pixel (lx, ly) becomes v' = saturate_u8(rint(float32(v) g)) in float32, g = the map's
 *   bilinear resize to the ROI at (lx, ly) (udh_gain_map: the taps of every ROI column and row, the row pass then the column
 *   pass, each product and sum rounded to float32; channel c's gain, or the one gain when channels = 1). */
#define UDH_EXPOSURE_MAX_BLOCKS (1 << 24)
size_t udh_mosaic_exposure_block_workspace_bytes(int n);
int udh_mosaic_exposure_block_stats_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const int32_t* rois, int n,
                                       const int32_t* blocks, const int64_t* boff, int64_t nblocks, const int32_t* pair_ptr,
                                       const int32_t* pair_j, int npairs, const int64_t* cell_off, const int32_t* cell_nx,
                                       int64_t nslots, const double* history, int feeds, int norms, int dst_h, int dst_w,
                                       uint64_t* stats, void* ws, size_t ws_bytes, void* stream);
size_t udh_exposure_block_solve_workspace_bytes(int n);
int udh_exposure_block_solve(int n, const int32_t* row_ptr, const int32_t* col, const double* val, const double* b, double tol,
                             int max_iter, double* x, int64_t* info, void* ws, size_t ws_bytes, void* stream);
size_t udh_exposure_gain_maps_workspace_bytes(int64_t nblocks, int channels);
int udh_exposure_gain_maps(const double* gains, int n, const int32_t* blocks, const int64_t* boff, int64_t nblocks, int channels,
                           float* maps, void* ws, size_t ws_bytes, void* stream);

/* ---- seam finding (cv2.detail's Voronoi seam finder; oracle/seam.py restates the rule) -------------------------------
 * udh_mosaic_seam_masks_u8: the seams between udh_mosaic_multiband_u8's frames (frames, sizes, M frame -> ROI (device),
 *   rois (host), as that call takes them), byte for byte what cv2.detail.SeamFinder_createDefault(VORONOI_SEAM).find
 *   leaves in their validity masks.  Each frame's mask starts as its ROI warp's validity (255 / 0).  Then, for every pair
 *   in the CSR list pair_ptr [n + 1], pair_j (host int32; row i, ascending j > i; the pairs must have intersecting ROIs;
 *   list every such pair for cv2's result), in that order, on the masks as the earlier pairs left them: over the ROIs'
 *   intersection grown by 10 px (s_i: frame i's mask inside its ROI, 0 outside), d_i is the exact L1 distance to the
 *   nearest pixel held by frame i alone (infinite if there is none), likewise d_j; over the intersection, frame j's mask
 *   is cleared where d_i < d_j and frame i's elsewhere.  seam [sum of roi_h roi_w] uint8 (device) receives the masks,
 *   frame k's rh x rw bytes at offset sum_{l<k} roi_h_l roi_w_l; blend (same layout) the blend masks cv2's stitcher feeds
 *   its blender: the 3 x 3 dilation of the seam mask AND the validity.  Launches 2 + 2 (pairs).  n <= UDH_SEAM_MAX_FRAMES,
 *   sides < 32767.  ws: udh_mosaic_seam_workspace_bytes(rois, n, pair_ptr, pair_j, dst_h, dst_w) bytes of device memory
 *   (0: bad arguments). */
#define UDH_SEAM_MAX_FRAMES 1024
size_t udh_mosaic_seam_workspace_bytes(const int32_t* rois, int n, const int32_t* pair_ptr, const int32_t* pair_j, int dst_h,
                                       int dst_w);
int udh_mosaic_seam_masks_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const int32_t* rois, int n,
                             const int32_t* pair_ptr, const int32_t* pair_j, int dst_h, int dst_w, uint8_t* seam, uint8_t* blend,
                             void* ws, size_t ws_bytes, void* stream);

/* udh_mosaic_seam_gc_masks_u8: the same call with cv2.detail's GraphCutSeamFinder(COST_COLOR) rule (oracle/seam_gc.py):
 *   the pairs, the window, s_i and s_j as above; I_i is frame i's ROI warp where the window pixel lies inside its ROI (its
 *   border values included), 0 outside, likewise I_j, and d = sum_c (I_i - I_j)^2.  The window is a 4-connected graph:
 *   edge (p, q) carries d(p) + d(q) + 1 both ways, + 1000 unless s_i and s_j hold both p and q; a pixel with s_i and not
 *   s_j is tied to the source, one with s_j and not s_i to the sink, with 10000.  T is the set of pixels that reach the
 *   sink in the residual graph of a maximum flow (the same for every maximum flow), S the rest; over the intersection,
 *   frame j's mask is cleared where p is in S and frame i holds it, frame i's where p is in T and frame j holds it.
 *   cut (host, optional): npairs int64, each pair's minimum-cut value.  Synchronises; the launches depend on how fast each
 *   pair's flow settles.  ws: udh_mosaic_seam_gc_workspace_bytes(rois, n, pair_ptr, pair_j, dst_h, dst_w) bytes of device
 *   memory (0: bad arguments).
 * udh_debug_grid_mincut: the minimum cut of an h x w grid graph (device int32 planes [h,w]): hcap[y,x] the capacity of
 *   edge (x, y) - (x + 1, y) both ways (last column ignored), vcap[y,x] of (x, y) - (x, y + 1) (last row ignored), src and
 *   snk the terminal capacities; every one in [0, 2^24].  T [h,w] uint8 (device): 1 where the pixel reaches the sink in
 *   the residual graph of a maximum preflow, 0 elsewhere; *cut (host): the cut's capacity; residual (device, optional)
 *   int32 [5,h,w]: the residual capacities to the right, lower, left and upper neighbour and to the sink.  Synchronises.
 *   ws: udh_debug_grid_mincut_workspace_bytes(h, w) bytes (0: sides outside 1..32786). */
size_t udh_mosaic_seam_gc_workspace_bytes(const int32_t* rois, int n, const int32_t* pair_ptr, const int32_t* pair_j, int dst_h,
                                          int dst_w);
int udh_mosaic_seam_gc_masks_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const int32_t* rois, int n,
                                const int32_t* pair_ptr, const int32_t* pair_j, int dst_h, int dst_w, uint8_t* seam, uint8_t* blend,
                                int64_t* cut, void* ws, size_t ws_bytes, void* stream);
size_t udh_debug_grid_mincut_workspace_bytes(int h, int w);
/* ---- seams at a reduced resolution (cv2's seam_megapix; oracle/seam_scale.py restates the rule) -----------------------
 * udh_resize_linear_exact_u8: cv2.resize(src, ..., INTER_LINEAR_EXACT) on n uint8 [src_h,src_w,c] images (c = 1 or 3),
 *   byte for byte, down or up.  tab (device, int32; ops.linear_exact_table): xs0[dst_w], xs1[dst_w], xc1[dst_w],
 *   ys0[dst_h], ys1[dst_h], yc1[dst_h]: per output column / row its two source taps and the upper tap's weight in 1/256
 *   (f = (d + 1/2) scale - 1/2 in float64, c1 = rint((f - floor f) 256), taps clamped to the image); each value is
 *   (c0' (c0 p00 + c1 p01) + c1' (c0 p10 + c1 p11) + 2^15) >> 16.  n <= 65535, dst_h dst_w < 2^31.
 * udh_mosaic_seam_upscale_u8: the full-resolution blend masks of seams found at scale (0, 1]: frames, sizes, M frame ->
 *   ROI (device) and rois (host) as udh_mosaic_seam_masks_u8 takes them (every ROI non-empty); seams [n] (device) frame
 *   k's seam mask on its seam ROI seam_rois[k] (host int32 [n,4] on the seam_h x seam_w seam canvas; an empty rectangle
 *   gives an all-zero mask and its pointer is ignored).  blend [sum of roi_h roi_w] (device, udh_mosaic_seam_masks_u8's
 *   layout) receives, at each ROI pixel (canvas X, Y), the frame's validity (0 / 255) AND the INTER_LINEAR_EXACT sample
 *   at ((X + 1/2) scale - 1/2, (Y + 1/2) scale - 1/2) of cv2.dilate(seam mask) placed on the seam canvas (0 outside its
 *   seam ROI), the taps built on the host in float64 and clamped to the seam canvas: graded masks, 1 .. 254 along the
 *   seams.  Launches 2 (1 when no seam ROI is given).  ws: udh_mosaic_seam_upscale_workspace_bytes(rois, seam_rois, n,
 *   seam_h, seam_w, scale, dst_h, dst_w) bytes of device memory (0: bad arguments). */
int udh_resize_linear_exact_u8(const uint8_t* src, const int32_t* tab, uint8_t* dst, int n, int src_h, int src_w, int c, int dst_h,
                               int dst_w, void* stream);
size_t udh_mosaic_seam_upscale_workspace_bytes(const int32_t* rois, const int32_t* seam_rois, int n, int seam_h, int seam_w,
                                               double scale, int dst_h, int dst_w);
int udh_mosaic_seam_upscale_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const int32_t* rois,
                               const uint8_t* const* seams, const int32_t* seam_rois, int n, int seam_h, int seam_w, double scale,
                               int dst_h, int dst_w, uint8_t* blend, void* ws, size_t ws_bytes, void* stream);
int udh_debug_grid_mincut(const int32_t* hcap, const int32_t* vcap, const int32_t* src, const int32_t* snk, int h, int w, uint8_t* T,
                          int64_t* cut, int32_t* residual, void* ws, size_t ws_bytes, void* stream);

/* ---- instrumentation read by bench.py -------------------------------------------------------------------------
 * udh_launch_count: kernels this library has launched in this process (monotonic).
 * udh_prof_*: when enabled, every tagged phase is bracketed by CUDA events recorded on the launching stream;
 * udh_prof_read synchronises on them and returns the accumulated device time and the number of brackets.
 * Must be off while a stream is being captured into a CUDA graph. */
unsigned long long udh_launch_count(void);
/* Leave n SMs free in the persistent one-CTA-per-SM tensor-core kernels (process-wide).  Used in data-parallel runs so
 * that the NCCL allreduce kernel overlapping the backward gets its own SMs instead of displacing persistent CTAs (a
 * displaced CTA would only start after another one finishes, i.e. serialise its whole share of the work). */
int udh_set_sm_reserve(int n);
/* Same, but only for the backward kernels of conv4_1 / conv4_2 (the launches that run while the fully connected gradients
 * are being all-reduced on the communication stream).  A persistent kernel with a static item schedule that finds n of its
 * SMs taken by the NCCL kernel runs those CTAs in a second wave (2x its time); with <= 2 items per CTA these four launches
 * lose nothing by starting on (SMs - n) CTAs, so reserving NCCL's CTA count here removes the collision. */
int udh_set_sm_reserve_top(int n);
/* CTAs (of 256 threads) of the Adam launches that follow; 0 = the default, enough to fill the device.  An update that runs
 * on a second stream underneath the conv backward is given one or two CTAs per SM so that the persistent tensor-core CTAs
 * (one per SM, ~200 KB of shared memory, <= 256 threads) stay co-resident with it instead of queueing behind it. */
int udh_set_adam_grid(int blocks);
/* A point inside the conv backward for a second stream to start at: with layer = 7..0 (conv4_2..conv1_1; -1 = off) every
 * conv backward that follows records an internal event on its stream right before the backward kernels of that layer, and
 * udh_bwd_marker_wait(stream) makes `stream` wait for the most recent record (no-op before the first).  The engine uses it
 * to run the fused gradient-reduce / Adam / weight-multicast kernel under the wide 64-channel layers' backward (tensor-bound)
 * rather than under conv4_x / conv3_x (short, latency-bound launches that a co-running streaming kernel slows 3-5x). */
int udh_set_bwd_marker(int layer);
/* SMs the persistent backward kernels of the marker layer and of the layers below it leave free (0 = none): a kernel of
 * 200+ KB of shared memory per CTA cannot share an SM with anything, so the second stream's kernel gets SMs of its own for
 * the length of that window and is launched with exactly that many CTAs. */
int udh_set_sm_reserve_marker(int n);
int udh_bwd_marker_wait(void* stream);

/* Row G + the optimiser for ONE rank's shard of a replicated tensor, over NVSwitch multicast memory (csrc/dp_update.cu):
 * replaces, for fc1's weights, code/utils/utils.py:380-403 (gradient mean over the towers) followed by
 * code/homography_CNN_synthetic.py:277-284 (apply_gradients).  mc_grads / mc_params are the MULTICAST addresses of the
 * flat gradient / parameter buffers (symmetric allocations bound to one multicast object; the same float offsets as the
 * local buffers), params / adam_m / adam_v the rank's local flat buffers.  For the floats [shard_begin, shard_begin +
 * shard_count): g = sum over ranks (multimem.ld_reduce) * grad_scale; TF-1 Adam on the local m, v; the new fp32 value is
 * stored to every replica (multimem.st), and so are its tensor-core limbs when mc_mirror (multicast address of the fc1
 * weight mirror, udh_cnn_fc1_mirror; planes of mirror_count elements, hi then lo) is given: mirror_limbs = 1 (bf16) or 2
 * (bf16x3), 0 with mc_mirror == NULL.  The gradient itself is left as is (fc1's weight gradient is stored, not accumulated).
 * The caller orders the ranks: every rank's gradient must be final before any rank launches this, and every rank's launch
 * must have completed before any replica is read (two symmetric-memory barriers on the stream, engine.py).  grid = CTAs of
 * 512 threads (0 = one per SM). */
int udh_dp_shard_update(const void* mc_grads, const float* params, void* mc_params, float* adam_m, float* adam_v,
                        void* mc_mirror, size_t shard_begin, size_t shard_count, size_t mirror_begin, size_t mirror_count,
                        int mirror_limbs, float alpha_t, float beta1, float beta2, float eps, float grad_scale, int grid,
                        void* stream);
/* HOST function (no device work): CRC-32C (Castagnoli) of n bytes, continuing from `crc` (0 to start) — the checksum of
 * TensorFlow checkpoint V2 bundles (tf.train.Saver, code/homography_CNN_synthetic.py:303,360), which tf_checkpoint.py writes
 * and verifies.  Hardware crc32 instruction when the CPU has SSE4.2, slicing-by-8 otherwise. */
uint32_t udh_crc32c(const void* data, size_t n, uint32_t crc);
int udh_prof_enable(int on);
int udh_prof_reset(void);
int udh_prof_num_tags(void);
const char* udh_prof_tag_name(int tag);
int udh_prof_read(int tag, float* total_ms, int* count);

/* ---- debug / test entry points of the tensor-core path ---------------------------------------------------------
 * udh_debug_tc_conv: ONE wgmma 3x3 convolution on fp32 NHWC tensors (pads + casts to bf16 internally), so tests can
 * compare the tensor-core kernel with a reference convolution layer by layer; dgrad != 0 runs the mirrored kernel. */
size_t udh_debug_tc_conv_scratch_bytes(int B, int H, int W, int cin, int cout);
int udh_debug_tc_conv(const float* x, const float* w, const float* bias, float* out, void* scratch, int B, int H, int W,
                      int cin, int cout, int relu, int dgrad, void* stream);
/* tensor-core weight gradient of one layer: x [B,H,W,cin], g [B,H,W,cout] fp32 -> dW HWIO, db (both accumulated);
 * scratch sized by udh_debug_tc_conv_scratch_bytes. */
int udh_debug_tc_wgrad(const float* x, const float* g, float* dW, float* db, void* scratch, int B, int H, int W, int cin,
                       int cout, void* stream);
/* UDH_NUMERIC_BF16X3 kernels, one layer at a time on fp32 NHWC tensors (split into limbs internally): 3x3 convolution
 * (forward or mirrored), weight gradient, and conv1_1 (forward when out != NULL, weight gradient when g != NULL). */
/* UDH_NUMERIC_BF16X3 workspace: write fp32 copies (hi + lo) of the saved conv / pool activations into the slots
 * udh_cnn_activation names; *fp32_region_bytes (nullable) = size of the leading part of the workspace whose layout is common
 * to all numeric modes (activations, dropout masks, fc buffers), so a test can run the fp32 backward on this forward state. */
int udh_debug_x3_materialize(void* ws, size_t ws_bytes, int B, int P, size_t* fp32_region_bytes, void* stream);
/* conv1_2 of the UDH_NUMERIC_BF16X3 mode runs on row tiles by default (forward fused with pool1: the full-resolution
 * activation is never stored; row-tile dgrad).  on = 0 selects the generic flattened-tile kernels + the separate pool kernel —
 * tests compare the two paths and need the un-fused one to read conv1_2's activation. */
int udh_debug_x3_set_rows(int on);
size_t udh_debug_x3_scratch_bytes(int B, int H, int W, int cin, int cout);
int udh_debug_x3_conv(const float* x, const float* w, const float* bias, float* out, void* scratch, int B, int H, int W, int cin,
                      int cout, int relu, int dgrad, void* stream);
/* udh_debug_x3_conv with the fused ReLU-mask epilogues of the train step.  Both masks are uint32 words over the PADDED
 * positions q = (n (H+2) + y + 1) (W+2) + x + 1 of the output, kout / 32 words per position (kout = cout, or cin when
 * dgrad != 0): bit j of word k of position q is channel 32k + j.  mask_bits (nullable, in) zeroes every output element whose
 * bit is clear (after bias and ReLU); mask_out (nullable, out, B (H+2) (W+2) kout / 32 words) receives out > 0, with zero
 * words at border positions. */
int udh_debug_x3_conv_ex(const float* x, const float* w, const float* bias, const uint32_t* mask_bits, uint32_t* mask_out,
                         float* out, void* scratch, int B, int H, int W, int cin, int cout, int relu, int dgrad, void* stream);
/* conv1_2's row-tile kernels (64 -> 64 channels, W == 128, even H), as the train step runs them:
 *   rows = 1: forward + bias + ReLU fused with the 2x2 max-pool; x [B,H,128,64] -> out = pooled [B,H/2,64,64] fp32 and
 *             codes [B,H/2,64,8] uint32 (3 bits per channel at (c % 8) * 3 of word c / 8: window index 0-3 of the maximum in
 *             row-major order, 4 where the maximum is not positive); bias and codes are required;
 *   rows = 2: dgrad (mirrored weights, no bias) of g [B,H,128,64] with the mask words of udh_debug_x3_conv_ex fused
 *             (mask_bits nullable); out [B,H,128,64]; codes is ignored.
 * scratch: udh_debug_x3_scratch_bytes(B, H, W, 64, 64). */
int udh_debug_x3_conv_rows(const float* x, const float* w, const float* bias, const uint32_t* mask_bits, float* out, uint32_t* codes,
                           void* scratch, int B, int H, int W, int rows, void* stream);
int udh_debug_x3_wgrad(const float* x, const float* g, float* dW, float* db, void* scratch, int B, int H, int W, int cin, int cout,
                       void* stream);
int udh_debug_x3_conv1(const float* I1, const float* I2, const float* w, const float* bias, float* out, const float* g, float* dW,
                       float* db, void* scratch, int B, int H, int W, void* stream);
/* udh_debug_x3_conv1 with conv1_1's fused ReLU-mask epilogue of the train step: mask_out (nullable; needs out) receives
 * out > 0 as the uint32 words of udh_debug_x3_conv_ex over the padded positions (2 words per position); the words of border
 * positions are not written. */
int udh_debug_x3_conv1_ex(const float* I1, const float* I2, const float* w, const float* bias, uint32_t* mask_out, float* out,
                          const float* g, float* dW, float* db, void* scratch, int B, int H, int W, void* stream);
/* fused conv (64 -> 64 channels, W == 128) + bias + ReLU + 2x2 max-pool (conv1_2 + pool1): x [B,H,128,64] ->
 * pooled [B,H/2,64,64] fp32 and routing codes [B,H/2,64,8] uint32 (3 bits per channel, 4 = no gradient). */
int udh_debug_tc_conv_pool(const float* x, const float* w, const float* bias, float* pooled, uint32_t* codes, void* scratch,
                           int B, int H, int W, void* stream);
/* the 2x2 max-pool kernels the step runs in numeric_mode UDH_NUMERIC_BF16X3 (pool_fwd_x3 / pool_bwd_x3) or UDH_NUMERIC_BF16
 * (pool_fwd_bf16 / pool_bwd_bf16), on fp32 NHWC tensors through the step's padded streams (two-limb split, or bf16 rounding).
 * Forward when in != NULL: in [B,H,W,C] -> out [B,H/2,W/2,C] (the stored pooled value, read back as fp32) and codes
 * [B,H/2,W/2,C/8] uint32 (3 bits per channel at (c % 8) * 3 of word c / 8: window index 0-3 of the first maximum in row-major
 * order, 4 where the maximum is not positive).  Backward when din != NULL: codes + dout [B,H/2,W/2,C] -> din [B,H,W,C] (the
 * stored gradient at the routed element, 0 elsewhere); a call with both runs the forward first.  H, W even, C % 8 == 0.  The
 * streams are allocated on `stream` and freed behind the kernels. */
int udh_debug_tc_pool(int numeric_mode, const float* in, float* out, uint32_t* codes, const float* dout, float* din, int B, int H,
                      int W, int C, void* stream);
/* fc1 (32768 -> 1024, the 128x128-patch regressor) through exactly the calls the step makes in `numeric_mode`:
 * y[B,1024] = x[B,32768] . w[32768,1024] (no bias, no ReLU); with dy[B,1024] != NULL also dW[32768,1024] = x^T . dy and
 * dx[B,32768] = dy . w^T, computed from the operand copies the forward made.  dW is STORED in the tensor-core modes and
 * ACCUMULATED in UDH_NUMERIC_FP32, as in the step.  scratch: udh_debug_fc1_scratch_bytes(B, numeric_mode) bytes (0 and
 * unused in UDH_NUMERIC_FP32; 0 also for B < 1 or an unknown mode); it receives, each at a 256-byte aligned offset, the
 * 16-bit copies of x [B][32768 x limbs], w (fc1's weight mirror: bf16, or the hi plane then the lo plane in
 * UDH_NUMERIC_BF16X3) and dy, which the forward casts from w itself (the step's mirror is not assumed current). */
size_t udh_debug_fc1_scratch_bytes(int B, int numeric_mode);
int udh_debug_fc1(int numeric_mode, const float* x, const float* w, const float* dy, float* y, float* dW, float* dx, void* scratch,
                  int B, void* stream);
/* fc1 of the P x P-patch regressor in UDH_NUMERIC_FP32 (the only mode above P = 128), F = (P/8)^2 * 128 features, through
 * exactly the calls the step makes: y[B,1024] = x[B,F] . w[F,1024] (split-K, no bias, no ReLU); with dy[B,1024] != NULL also
 * dW[F,1024] += x^T . dy (ACCUMULATED, as in the step) and dx[B,F] = dy . w^T.  B and P are checked as udh_cnn_fwd checks
 * them (P a multiple of 128 up to 1408).  All buffers are the caller's. */
int udh_debug_fc1_ex(const float* x, const float* w, const float* dy, float* y, float* dW, float* dx, int B, int P, void* stream);

/* ---- debug / test entry points of the fp32 CUDA-core path (UDH_NUMERIC_FP32), the calls the step makes ------------
 * udh_debug_simt_conv: one 3x3 convolution, NHWC fp32, H % 8 == 0, W % 16 == 0.  dgrad == 0: out [B,H,W,cout] =
 * relu?(conv(x, w) + bias) (bias nullable), with x2 != NULL the two single-channel planes x, x2 of conv1_1 (cin == 2).
 * dgrad != 0: w is the layer's [3,3,cin,cout] kernel; it is rotated into wrot (9 cin cout floats) and out [B,H,W,cin] =
 * conv(x = g [B,H,W,cout], wrot) with no bias, no ReLU and no second plane.  mask_src (nullable, shaped like out) zeroes
 * every output element whose mask_src value is not > 0 (the fused ReLU backward of the layer below). */
int udh_debug_simt_conv(const float* x, const float* x2, const float* w, const float* bias, const float* mask_src, float* out,
                        float* wrot, int B, int H, int W, int cin, int cout, int relu, int dgrad, void* stream);
/* weight gradient of one layer: dW [3,3,cin,cout] += sum x * g and db [cout] += sum g (fp32 atomics: not bit-reproducible),
 * x [B,H,W,cin] (or the planes x, x2 with cin == 2), g [B,H,W,cout].  The partition (nullable outputs): CTA x (of ctas_x)
 * walks pixel tiles [x tiles_per_cta, (x+1) tiles_per_cta) of the B (H/8) (W/16) 8x16 tiles in (n, tile row, tile column)
 * order; its threads for rows s = 0 .. row_split-1 each sum rows s, s + row_split, ... of those tiles, in order of tile, row
 * and column, with one fmaf per pixel, and add their partial to dW with one atomicAdd (db likewise with plain adds). */
int udh_debug_simt_wgrad(const float* x, const float* x2, const float* g, float* dW, float* db, int B, int H, int W, int cin,
                         int cout, int* ctas_x, int* tiles_per_cta, int* row_split, void* stream);
/* 2x2 max-pool of in [B,H,W,C]: forward into out [B,H/2,W/2,C] when out != NULL; backward when din != NULL: din [B,H,W,C]
 * receives dout [B,H/2,W/2,C] at the first maximum of each window in row-major order when that maximum is > 0, else 0. */
int udh_debug_simt_pool(const float* in, float* out, const float* dout, float* din, int B, int H, int W, int C, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* UDH_H_ */
