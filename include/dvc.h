/*
 * libdvc.so -- C ABI of the H100-native exemplar-video-colorization forward path.
 *
 * The reference (zhangmozhe/Deep-Exemplar-based-Video-Colorization) has no FFI of its own: its
 * hot path is three Python nn.Module.forward() methods plus per-frame glue.  Each entry point below
 * names the reference interface it replaces (file:line relative to the reference root).  The
 * Python drop-in modules (models/NonlocalNet.py, models/ColorVidNet.py in the package) bind these
 * symbols with ctypes; INTEGRATION.md shows that binding.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross the boundary.
 *   - tensors are fp32, contiguous, NCHW unless stated; `dev_*` pointers are device memory on the
 *     context's device, `host_*` pointers are host memory (pinned for the async paths).
 *   - every function returns DVC_OK (0) or a negative dvc_status; dvc_last_error() gives the text.
 *   - all device work is enqueued on the `stream` argument (a cudaStream_t passed as void*); no
 *     entry point synchronises the device unless stated.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with
 *     DVC_ERR_CUDA.
 *   - legal frame shapes are the reference's (SURVEY.md fact 2): H % 8 == 0, W % 16 == 0, H,W >= 32;
 *     anything else returns DVC_ERR_SHAPE before any launch (the reference raises RuntimeError at
 *     NonlocalNet.py:464, or at VGG19's fifth max-pool when the r52 map is narrower than 2x2).
 */
#ifndef DVC_H_
#define DVC_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dvc_ctx dvc_ctx;

typedef enum dvc_status {
  DVC_OK = 0,
  DVC_ERR_ARG = -1,     /* null pointer, unknown key, unsupported option (pool="avg", WTA_scale_weight != 1) */
  DVC_ERR_SHAPE = -2,   /* illegal H/W or mismatching tensor shape */
  DVC_ERR_CUDA = -3,    /* CUDA runtime error (text in dvc_last_error) or no device */
  DVC_ERR_STATE = -4,   /* weights missing, exemplar not set, ... */
  DVC_ERR_NCCL = -5
} dvc_status;

typedef enum dvc_net { DVC_NET_VGG = 0, DVC_NET_WARP = 1, DVC_NET_COLOR = 2 } dvc_net;

/* Arithmetic used by the GEMM-shaped kernels (convolutions, correlation).
 *   DVC_MATH_FP32    CUDA-core fp32 FMA (exact fp32 products, two-level accumulation; the on-GPU fp32 reference)
 *   DVC_MATH_TF32X3  wgmma tf32 on hi/lo split operands, 3 MMAs per product, accumulator chunk sums promoted
 *                    to fp32 registers (fp32-class accuracy; THE DEFAULT for convolutions and correlation)
 *   DVC_MATH_BF16X3  wgmma bf16 on hi/lo split operands (correlation only; fast mode, |df| ~ 2e-6)
 *   DVC_MATH_FP16X3  wgmma fp16 on hi/lo planes of x * 2^14 (correlation only: its operands are unit
 *                    vectors, so the power-of-two scale is exact): tf32x3's 2 x 11 bits at bf16x3's speed
 *   DVC_MATH_FP16X1  convolutions only, opt-in fast mode: ONE MMA per product, hi * hi, on the operand planes of
 *                    DVC_MATH_TF32X3 -- an fp16 wgmma on the fp16 planes of x * 2^e_x and w * 2^e_w (exact
 *                    power-of-two scales), a tf32 wgmma on the tf32 planes of inputs without a known bound.  Every
 *                    conv operand is thus rounded to 11 significant bits (round-to-nearest), as PyTorch's cuDNN
 *                    convolutions round fp32 operands to TF32 by default (torch.backends.cudnn.allow_tf32); the
 *                    products are exact and summed as in TF32X3.  Error per output <= ~2^-10 * sum |x| |w|.
 *                    Activations, InstanceNorm, the small first layers and the correlation keep the default
 *                    arithmetic.  Not accepted as corr_math (DVC_ERR_ARG).
 */
typedef enum dvc_math {
  DVC_MATH_FP32 = 0,
  DVC_MATH_TF32X3 = 1,
  DVC_MATH_BF16X3 = 2,
  DVC_MATH_FP16X3 = 3,
  DVC_MATH_FP16X1 = 4
} dvc_math;

/* ---- lifetime ------------------------------------------------------------------------------- */

/* One context per device (reference: test.py:147-166 builds one set of modules on cuda:0).
 * Not thread-safe per context. */
int dvc_create(dvc_ctx** out, int device);
int dvc_destroy(dvc_ctx* ctx);
const char* dvc_last_error(const dvc_ctx* ctx); /* ctx may be NULL: last create() error */
const char* dvc_version(void);

/* Select the arithmetic of the conv layers (FP32, TF32X3, FP16X1) and of the correlation (FP32, TF32X3, BF16X3,
 * FP16X3; see dvc_math).  Both are validated before anything changes: a refused call leaves the context as it was.
 * A change of conv_math invalidates the cached exemplar(s): set them again. */
int dvc_set_math(dvc_ctx* ctx, int conv_math, int corr_math);

/* ---- weights: replaces nn.Module.load_state_dict (test.py:150,158-159) ----------------------- */

/* `data` holds the tensor for `key` exactly as in the reference state_dict (OIHW fp32 for conv
 * weights, [C] for biases, [1] for PReLU slopes, [C,1,1,1] for the depthwise *_ss scales).
 * `data` may be a host or a device pointer (cudaMemcpyDefault).  Synchronous. */
int dvc_set_weight(dvc_ctx* ctx, int net, const char* key, const float* data, const int64_t* shape, int ndim);

/* ---- module-level drop-ins ------------------------------------------------------------------ */

/* VGG19_pytorch.forward(x, out_keys, preprocess) -- models/NonlocalNet.py:228-256.
 * dev_x [B,3,H,W] RGB in [0,1].  keys[i] in {"r11".."r54","p1".."p5"}; dev_out[i] receives that map
 * (NCHW fp32, caller-allocated).  Like the reference, preprocess != 0 applies util.py:347-352. */
int dvc_vgg19_forward(dvc_ctx* ctx, const float* dev_x, int B, int H, int W, int preprocess,
                      const char* const* keys, float* const* dev_out, int n_keys, void* stream);

/* WarpNet.forward(B_lab_map, A_relu2_1..5_1, B_relu2_1..5_1, temperature, ...) --
 * models/NonlocalNet.py:427-502.  dev_A[4]/dev_Bf[4] are the (already feature_normalize()d) r22,r32,r42,r52
 * maps: [B,128,H/2,W/2], [B,256,H/4,W/4], [B,512,H/8,W/8], [B,512,H/16,W/16].
 * dev_y [B,3,H,W], dev_sim [B,1,H,W].  reuse_exemplar != 0 skips the B-side recomputation and uses the
 * phi / pooled-Lab operands cached by the previous call (valid only for identical B tensors).
 * wta_scale_weight must be 1 (the reference bypasses WTA_scale in that case, NonlocalNet.py:486). */
int dvc_warpnet_forward(dvc_ctx* ctx, const float* dev_B_lab_map, const float* const* dev_A,
                        const float* const* dev_Bf, int B, int H, int W, float temperature,
                        float wta_scale_weight, int reuse_exemplar, float* dev_y, float* dev_sim, void* stream);

/* ColorVidNet.forward(x) -- models/ColorVidNet.py:96-144.  dev_x [B,7,H,W] -> dev_out [B,2,H,W]. */
int dvc_colorvidnet_forward(dvc_ctx* ctx, const float* dev_x, int B, int H, int W, float* dev_out, void* stream);

/* ---- the correlation kernel on its own (microbench / unit-test entry) ------------------------ */

/* f = theta_hat^T phi_hat; sim = rowmax f; P = softmax_j(f/T); y = P V   (NonlocalNet.py:477-498)
 * dev_theta_hat [B,C,NA], dev_phi_hat [Bphi,C,NB] (Bphi == B or 1: one exemplar shared by B frames),
 * dev_V [Bphi,NB,3]; outputs dev_y [B,NA,3], dev_sim [B,NA]; dev_argmax [B,NA] int32 may be NULL.
 * C must be a multiple of 64 (256 = WarpNet.inter_channels, NonlocalNet.py:360; other depths, e.g. the patch features of
 * NonlocalWeightedAverage, NonlocalNet.py:95-108, take the exact 3-pass kernel). */
int dvc_corr_softmax_warp(dvc_ctx* ctx, const float* dev_theta_hat, const float* dev_phi_hat,
                          const float* dev_V, int B, int Bphi, int NA, int NB, int C, float temperature,
                          float* dev_y, float* dev_sim, int32_t* dev_argmax, void* stream);
/* One query set against K reference sets (1 <= K <= 8; the correlation of dvc_colorize_frames_exemplars): theta_hat
 * [1,C,NA], phi_hat [K,C,NB], V [K,NB,3] -> y [K,NA,3], sim [K,NA], argmax [K,NA] (may be NULL).  Slot k equals
 * dvc_corr_softmax_warp(theta_hat, phi_hat[k], V[k]) except for the summation order of softmax weights (T > 0) and of
 * the V rows of bit-equal maxima.  Not combined with peer outputs (dvc_corr_set_peer_outputs): DVC_ERR_STATE. */
int dvc_corr_softmax_warp_exemplars(dvc_ctx* ctx, const float* dev_theta_hat, const float* dev_phi_hat, const float* dev_V,
                                    int K, int NA, int NB, int C, float temperature, float* dev_y, float* dev_sim,
                                    int32_t* dev_argmax, void* stream);

/* ---- fused per-frame / per-clip path (test.py:57-96 + FrameColor.py:41-67) -------------------- */

/* Exemplar prologue, test.py:57-66: IB_lab [1,3,H,W] (centred L, a, b) -> sRGB -> VGG -> heads ->
 * phi_hat / pooled Lab, cached in the context.  Host or device pointer. */
int dvc_set_exemplar(dvc_ctx* ctx, const float* IB_lab, int H, int W, void* stream);

/* frame_colorization (FrameColor.py:41-67) for B frames against the cached exemplar.
 * IA_l [B,1,H,W] centred luminance; IA_last_lab [B,3,H,W]; out_ab [B,2,H,W];
 * optional out_warp_lab [B,3,H,W] and out_sim [B,1,H,W] (may be NULL).  All device pointers. */
int dvc_colorize_frames(dvc_ctx* ctx, const float* dev_IA_l, const float* dev_IA_last_lab, int B, int H, int W,
                        float temperature, float* dev_out_ab, float* dev_out_warp_lab, float* dev_out_sim,
                        void* stream);

/* A whole segment with the frame-to-frame recurrence of test.py:76-96 kept on the device:
 * host_L [F,1,H,W] (pinned) is copied in frame by frame, frame t's predicted ab feeds frame t+1,
 * host_ab [F,2,H,W] (pinned) receives the predictions.  first_last_lab: NULL = zeros (test.py:80) or a
 * host [1,3,H,W] tensor (test.py:78, --frame_propagate).  Synchronises `stream` before returning. */
int dvc_colorize_clip(dvc_ctx* ctx, const float* host_L, int F, int H, int W, float temperature,
                      const float* host_first_last_lab, float* host_ab, void* stream);

/* ---- several exemplars for one clip (test.py:168-181 colorizes the clip once per reference image) ------------
 * The half of every frame that does not depend on the exemplar (VGG19, feature_normalize, the WarpNet query side)
 * runs once; the correlation runs against all K cached exemplars and ColorVidNet at batch K.  Exemplar k's results
 * are those of frame_colorization(IA_t, IB_k, last_k) with last_k = cat(L_t, ab_k,t-1) (test.py:96): K independent
 * recurrences sharing one luminance sequence.  While K > 1 exemplars are cached, dvc_colorize_frames,
 * dvc_colorize_clip and dvc_exemplar_export return DVC_ERR_STATE; dvc_set_exemplar / dvc_exemplar_import cache one
 * again.  K outside [1, 8] is DVC_ERR_ARG, a K other than the cached count or a frame size other than the
 * exemplars' is DVC_ERR_SHAPE. */

/* K exemplars IB_lab [K,3,H,W] (host or device pointer): dvc_set_exemplar's prologue for each, cached in K slots (slot
 * k holds exactly what dvc_set_exemplar(IB_k) caches).  dvc_set_exemplar / dvc_exemplar_import are the K = 1 case. */
int dvc_set_exemplars(dvc_ctx* ctx, const float* IB_lab, int K, int H, int W, void* stream);
/* One frame against all K cached exemplars.  dev_IA_l [1,1,H,W]; dev_last_lab [K,3,H,W]; dev_out_ab [K,2,H,W];
 * optional dev_out_warp_lab [K,3,H,W] and dev_out_sim [K,1,H,W] (may be NULL).  K must equal the cached count. */
int dvc_colorize_frames_exemplars(dvc_ctx* ctx, const float* dev_IA_l, const float* dev_last_lab, int K, int H, int W,
                                  float temperature, float* dev_out_ab, float* dev_out_warp_lab, float* dev_out_sim,
                                  void* stream);
/* dvc_colorize_clip with K recurrences: L [F,1,H,W]; first_last_lab NULL (zeros, test.py:80) or [K,3,H,W]
 * (--frame_propagate, test.py:78); ab [K,F,2,H,W], so each exemplar's clip is contiguous.  Host (pinned) or device
 * memory, like dvc_colorize_clip.  Synchronises `stream` before returning. */
int dvc_colorize_clip_exemplars(dvc_ctx* ctx, const float* L, int F, int H, int W, float temperature,
                                const float* first_last_lab, int K, float* ab, void* stream);
/* test.py:68-120 end to end on the device, in one pipelined call: per frame of frames [F,Hs,Ws,3] (uint8 sRGB)
 *   CenterPad + CenterCrop (dvc_resize_antialias_crop_rgb8 with the geometry Hr, Wr, oy, ox, Ho, Wo, which the caller
 *   computes: dvc/prepost.py) -> centred L at Ho x Wo and at (Ho/2) x (Wo/2) (dvc_rgb8_to_lab's plane 0, dvc_resize_half;
 *   the frames' a / b are not computed) -> the networks against the K cached exemplars (dvc_colorize_clip /
 *   dvc_colorize_clip_exemplars; K = 1 after dvc_set_exemplar) -> ab x2 * 1.25 (dvc_upsample2_scaled) -> if wls, the
 *   Fast Global Smoother (wls_lambda, wls_sigma; lambda_attenuation 0.25, 3 iterations) of every a / b plane guided by
 *   dvc_l_to_guide8 of the full-resolution L -> dvc_lab_to_rgb8 with that L
 * into out [K,F,Ho,Wo,3] uint8.  The cached exemplar size must be (Ho/2, Wo/2); the output window must nest with the
 * resized image (0 <= oy <= Hr - Ho, or Hr - Ho <= oy <= 0; the same for x).  first_last_lab: NULL (zeros) or
 * [K,3,Ho/2,Wo/2]; last_lab_out: NULL or [K,3,Ho/2,Wo/2], receives cat(L/2, ab) of the last frame, so a clip cut into
 * segments, each continuing from the previous one's last_lab_out, gives the bytes of one call over the whole clip.
 * frames / out / first_last_lab / last_lab_out may be host (pinned) or device memory.  Device memory does not depend on
 * F.  Synchronises `stream` before returning; a refused call launches nothing. */
int dvc_colorize_video_rgb8(dvc_ctx* ctx, const unsigned char* frames, int F, int Hs, int Ws, int Hr, int Wr, int oy, int ox,
                            int Ho, int Wo, float temperature, const float* first_last_lab, int wls, float wls_lambda,
                            float wls_sigma, unsigned char* out, float* last_lab_out, void* stream);

/* ---- several clips in one pass, one exemplar each (a dataset or an archive: many independent runs of test.py:68-120) -----
 * Clip s is colorized against cached exemplar slot s (dvc_set_exemplars with S images; dvc_set_exemplar is S = 1) with its
 * own recurrence last_s = cat(L_s,t, ab_s,t) (test.py:96).  VGG19, the WarpNet query side and the correlation run at batch S
 * with frame s against slot s, ColorVidNet at batch S -- ColorVidNet is recurrent, so frames of other clips are what fills
 * its low-resolution layers.  All clips of a call share the frame size, the temperature and F; clips of different lengths
 * stream in chunks and leave between calls.  S = 1 gives the bits of the single-exemplar calls; with S > 1 a clip's results
 * equal its solo run up to the InstanceNorm summation order and the device-derived fp16 scales that ColorVidNet shares
 * across its batch.  S outside [1, 8] is DVC_ERR_ARG; an S other than the cached exemplar count or a frame size other than
 * the exemplars' is DVC_ERR_SHAPE.  A refused call launches nothing.  Several exemplars per clip: the *_clips_exemplars
 * entries below. */

/* dvc_colorize_frames for S frames, frame s against slot s: dev_IA_l [S,1,H,W]; dev_last_lab [S,3,H,W]; dev_out_ab [S,2,H,W];
 * optional dev_out_warp_lab [S,3,H,W] and dev_out_sim [S,1,H,W] (may be NULL).  All device pointers. */
int dvc_colorize_frames_clips(dvc_ctx* ctx, const float* dev_IA_l, const float* dev_last_lab, int S, int H, int W, float temperature,
                              float* dev_out_ab, float* dev_out_warp_lab, float* dev_out_sim, void* stream);
/* dvc_colorize_clip for S clips: L [S,F,1,H,W]; first_last_lab NULL (zeros) or [S,3,H,W]; ab [S,F,2,H,W].  Host (pinned)
 * or device memory.  Synchronises `stream` before returning. */
int dvc_colorize_clips(dvc_ctx* ctx, const float* L, int F, int H, int W, float temperature, const float* first_last_lab, int S,
                       float* ab, void* stream);
/* dvc_colorize_video_rgb8 for S clips: frames[s] points to clip s's [F,Hs_s,Ws_s,3] uint8 frames (the source sizes may differ
 * between clips); geom [S][6] holds (Hs, Ws, Hr, Wr, oy, ox) of each clip, each checked as dvc_colorize_video_rgb8 checks
 * its own; out [S,F,Ho,Wo,3]; first_last_lab and last_lab_out NULL or [S,3,Ho/2,Wo/2].  A null frames[s] is DVC_ERR_ARG.
 * Device memory does not depend on F.  Synchronises `stream` before returning. */
int dvc_colorize_videos_rgb8(dvc_ctx* ctx, int S, const unsigned char* const* frames, int F, const int* geom, int Ho, int Wo,
                             float temperature, const float* first_last_lab, int wls, float wls_lambda, float wls_sigma,
                             unsigned char* out, float* last_lab_out, void* stream);

/* ---- several clips in one pass, several exemplars each (the reference's data layout: a folder of reference images per
 * clip, each colorizing the whole clip, test.py:168-181) -------------------------------------------------------------------
 * Clip s has K[s] >= 1 exemplars; K points to the S per-clip counts.  A call works on R = K[0] + ... + K[S-1] rows: row r
 * is one (clip, exemplar) pair, the rows of clip s are contiguous and in its exemplar order (clip s's first row is
 * K[0] + ... + K[s-1]), and row r runs against cached exemplar slot r -- dvc_set_exemplars with the R images in row order.
 * VGG19 and the WarpNet query side run once per clip frame at batch S; the correlation of row r pairs its clip's query set
 * with slot r; ColorVidNet runs at batch R with each row's own recurrence last_r = cat(L_{clip of r},t, ab_r,t) (test.py:96).
 * All tensors are row-major over the R rows, so the layouts contain the existing ones: with S = 1, [R,...] is the [K,...] of
 * the *_exemplars calls, and with every K[s] = 1 the [S,...] of the several-clip calls -- whose bits these calls then give.
 * S outside [1, 8], a null K, any K[s] < 1 or R > 8 is DVC_ERR_ARG; an R other than the cached exemplar count or a frame size
 * other than the exemplars' is DVC_ERR_SHAPE.  A refused call launches nothing. */

/* frame s of dev_IA_l [S,1,H,W] against the K[s] slots of clip s: dev_last_lab [R,3,H,W]; dev_out_ab [R,2,H,W]; optional
 * dev_out_warp_lab [R,3,H,W] and dev_out_sim [R,1,H,W] (may be NULL).  All device pointers. */
int dvc_colorize_frames_clips_exemplars(dvc_ctx* ctx, const float* dev_IA_l, const float* dev_last_lab, int S, const int* K, int H,
                                        int W, float temperature, float* dev_out_ab, float* dev_out_warp_lab, float* dev_out_sim,
                                        void* stream);
/* dvc_colorize_clips with K[s] exemplars per clip: L [S,F,1,H,W]; first_last_lab NULL (zeros) or [R,3,H,W]; ab [R,F,2,H,W].
 * Host (pinned) or device memory.  Synchronises `stream` before returning. */
int dvc_colorize_clips_exemplars(dvc_ctx* ctx, const float* L, int F, int H, int W, float temperature, const float* first_last_lab,
                                 int S, const int* K, float* ab, void* stream);
/* dvc_colorize_videos_rgb8 with K[s] exemplars per clip: frames and geom as there; out [R,F,Ho,Wo,3]; first_last_lab and
 * last_lab_out NULL or [R,3,Ho/2,Wo/2].  The post-processing of row r (WLS guide, full-resolution L) is its clip's.  Device
 * memory does not depend on F.  Synchronises `stream` before returning. */
int dvc_colorize_videos_exemplars_rgb8(dvc_ctx* ctx, int S, const int* K, const unsigned char* const* frames, int F, const int* geom,
                                       int Ho, int Wo, float temperature, const float* first_last_lab, int wls, float wls_lambda,
                                       float wls_sigma, unsigned char* out, float* last_lab_out, void* stream);

/* ---- video output at the source resolution ---------------------------------------------------------------------------------
 * The networks run at the CenterPad window (Ho, Wo) = image_size; the reference leaves rescaling the output to the user.
 * These calls keep the source frame's own luminance and take only the chroma from the network: the window's ab (after x2 * 1.25)
 * is resampled bilinearly onto the source grid, WLS-filtered with the guide of the source frame's L and turned into sRGB with
 * that L -- test.py:100-119's recipe, run one grid further.  The output covers the footprint: the source pixels whose centres
 * fall inside the window's extent [-0.5, Ho - 0.5] x [-0.5, Wo - 0.5], i.e. the whole frame when the source has the window's
 * aspect ratio or the window zero-pads it, the centre band when CenterPad crops. */

/* Footprint of the window (Ho, Wo) on a source of geometry (Hs, Ws, Hr, Wr, oy, ox) (dvc_colorize_video_rgb8's): source row ys
 * is in it iff 2 oy Hs <= (2 ys + 1) Hr <= 2 (oy + Ho) Hs (exact integers; columns alike).  out[4] = (y0, x0, h, w).  Needs no
 * context or device.  DVC_ERR_ARG for a null out or a size < 1, DVC_ERR_SHAPE when no source pixel centre is inside. */
int dvc_source_footprint(int Hs, int Ws, int Hr, int Wr, int oy, int ox, int Ho, int Wo, int out[4]);
/* dev_ab [planes,Ho,Wo] (window grid) -> dev_dst [planes,h,w] on the footprint (y0, x0, h, w) of the source grid: pixel (ys, xs)
 * samples the window at cy = ((2 ys + 1) Hr - (2 oy + 1) Hs) / (2 Hs) (an exact integer numerator over one float64 division; cx
 * alike) clamped to [0, Ho - 1], bilinearly with dvc_upsample2_scaled's expression, every fp32 operation separately rounded.
 * With Hs = Hr = Ho and oy = 0 (ditto x) it is the identity. */
int dvc_ab_to_source(dvc_ctx* ctx, const float* dev_ab, int planes, int Ho, int Wo, int Hs, int Ws, int Hr, int Wr, int oy, int ox,
                     float* dev_dst, void* stream);
/* dvc_colorize_videos_exemplars_rgb8 (S clips, K[s] exemplars each; S = 1, K = (1) is the single-clip case) with every output
 * frame at its source resolution: out[s] points to clip s's own [K[s],F,h_s,w_s,3] uint8, (h_s, w_s) its footprint.  Per row:
 * the window ab -> dvc_ab_to_source -> if wls, the FGS of its a / b planes (wls_lambda, wls_sigma) guided by dvc_l_to_guide8 of the
 * source L -> dvc_lab_to_rgb8 with the source L, where the source L is dvc_rgb8_to_lab's plane 0 of the source frame over the
 * footprint.  lambda and sigma keep their per-pixel meaning: a 1080x1920 grid is 2.5x finer per axis than 432x768, so the
 * same lambda smooths over a 2.5x smaller fraction of the frame, and the caller may raise it.  The networks, the
 * recurrence, first_last_lab and last_lab_out are those of the window-size call ([R,3,Ho/2,Wo/2]), so chunked calls continue a
 * clip exactly.  Refuses what that call refuses, plus a null out or out[s], before any launch.  Device memory does not depend
 * on F.  Synchronises `stream` before returning. */
int dvc_colorize_videos_source_rgb8(dvc_ctx* ctx, int S, const int* K, const unsigned char* const* frames, int F, const int* geom,
                                    int Ho, int Wo, float temperature, const float* first_last_lab, int wls, float wls_lambda,
                                    float wls_sigma, unsigned char* const* out, float* last_lab_out, void* stream);

/* ---- JPEG output (test.py:120 writes every frame as a JPEG file) -------------------------------------------------------------
 * A baseline encoder on the device whose files are byte-identical to Pillow's Image.fromarray(x).save(f, "JPEG", quality=q)
 * with libjpeg-turbo: 4:2:0 YCbCr (jccolor.c, h2v2_downsample, edge replication), JDCT_ISLOW, jcdctmgr.c's quantizer, the
 * standard Huffman tables (optimize=False), no restart markers; markers SOI, APP0 JFIF 1.01, DQT luma, DQT chroma, SOF0, DHT
 * DC/AC luma, DC/AC chroma, SOS, the entropy-coded data, EOI.  Only the finished files leave the device.
 *
 * Upper bound on the file size of an H x W image for any content and any quality in [1, 100]:
 *   623 header bytes + 2 (EOI) + 2 * ceil(1660 * nblocks / 8),  nblocks = 6 ceil(H/16) ceil(W/16)
 * One block codes a DC difference (code <= 11 bits, value <= 11 bits: category <= 11) and 63 AC coefficients, each a code of
 * <= 16 bits (the longest standard code) and <= 10 value bits (category <= 10); a ZRL (<= 11 bits) stands for 16 zero
 * coefficients and an EOB (<= 4 bits) for >= 1, which would otherwise cost <= 26 bits each, so 22 + 63 * 26 = 1660 bits bound a
 * block; the final byte's 1-bit padding is within the ceil, and 0xFF 0x00 stuffing at most doubles the data.  Needs no context
 * or device.  DVC_ERR_SHAPE outside H, W in [1, 65535] or for 1660 * nblocks >= 2^31 (about 14 Mpixel). */
int64_t dvc_jpeg_max_bytes(int H, int W);
/* dev_rgb [B,H,W,3] uint8 (device) -> B JFIF files at quality `quality` in [1, 100] (jpeg_set_quality(q, force_baseline=TRUE)):
 * image b's file goes to out + b * stride, its length to sizes[b].  out and sizes may be device memory or page-locked host memory
 * (on unified addressing the kernels store into it directly, so only the written bytes cross PCIe); pageable host memory is
 * DVC_ERR_ARG, so are null pointers, B < 1 and a quality outside [1, 100]; stride < dvc_jpeg_max_bytes(H, W) is DVC_ERR_SHAPE.
 * Seven launches.  Asynchronous on `stream`: sizes and files are valid once it completes. */
int dvc_encode_jpeg(dvc_ctx* ctx, const unsigned char* dev_rgb, int B, int H, int W, int quality, unsigned char* out, int64_t stride,
                    int64_t* sizes, void* stream);
/* The frames of dvc_colorize_videos_exemplars_rgb8 (source_resolution = 0) or of dvc_colorize_videos_source_rgb8 (1), encoded as
 * dvc_encode_jpeg encodes them: out[s] holds clip s's [K[s],F] slots of `stride` bytes (row r_local of clip s, frame t at
 * out[s] + (r_local F + t) stride), sizes [R,F] their lengths.  The networks, the recurrence, first_last_lab and last_lab_out
 * are those of the rgb8 calls, so chunked calls continue a clip exactly.  The encoder runs on the post-processing stream after
 * Lab -> sRGB of each frame (7 launches per output size: one for the window, one per footprint size) and stores the finished
 * files straight into their slots; no per-frame host synchronisation, and device memory does not depend on F.  Refuses what the
 * underlying call refuses, a quality outside [1, 100] or a null out / out[s] / sizes (DVC_ERR_ARG), pageable host memory
 * (DVC_ERR_ARG) and a stride below dvc_jpeg_max_bytes of the largest output frame (DVC_ERR_SHAPE), before any launch.
 * Synchronises `stream` before returning. */
int dvc_colorize_videos_jpeg(dvc_ctx* ctx, int S, const int* K, const unsigned char* const* frames, int F, const int* geom, int Ho,
                             int Wo, float temperature, const float* first_last_lab, int wls, float wls_lambda, float wls_sigma,
                             int source_resolution, int quality, unsigned char* const* out, int64_t stride, int64_t* sizes,
                             float* last_lab_out, void* stream);

/* ---- greyscale sources -------------------------------------------------------------------------------------------------------
 * The video calls for single-channel frames: frames[s] is clip s's [F,Hs_s,Ws_s] uint8 (one byte per pixel), host-pinned or
 * device memory; K, geom, the rows, the recurrence, first_last_lab and last_lab_out are as in dvc_colorize_videos_exemplars_rgb8,
 * and exemplars stay colour images (dvc_set_exemplar(s)).
 *   quality == 0: out[s] receives clip s's sRGB frames [K[s],F,h,w,3], (h, w) the window (Ho, Wo), or the footprint
 *                 (dvc_source_footprint) when source_resolution is set; stride must be 0 and sizes NULL.
 *   quality in [1, 100]: out, stride and sizes are exactly dvc_colorize_videos_jpeg's.
 * Contract: every output byte (and, for JPEG, every size) and last_lab_out equal what the corresponding sRGB call --
 * dvc_colorize_videos_exemplars_rgb8 (with its [R,F,Ho,Wo,3] rows split by clip), dvc_colorize_videos_source_rgb8 or
 * dvc_colorize_videos_jpeg -- returns for the frames with each byte g replicated into (g, g, g).  Only Hs Ws bytes per frame
 * are uploaded and resized, and L is looked up per byte value; the launches per frame step are those of that call.  Refuses
 * what that call refuses, plus a null out / out[s], a quality outside [0, 100], and quality == 0 with a non-zero stride or a
 * non-null sizes (DVC_ERR_ARG), before any launch.  Synchronises `stream` before returning. */
int dvc_colorize_videos_gray8(dvc_ctx* ctx, int S, const int* K, const unsigned char* const* frames, int F, const int* geom, int Ho,
                              int Wo, float temperature, const float* first_last_lab, int wls, float wls_lambda, float wls_sigma,
                              int source_resolution, int quality, unsigned char* const* out, int64_t stride, int64_t* sizes,
                              float* last_lab_out, void* stream);

/* ---- planar YUV 4:2:0 (I420) video -----------------------------------------------------------------------------------------
 * The pixel format of video decoders and encoders (ffmpeg -pix_fmt yuv420p, x264, NVENC).  One H x W frame (H, W even) is
 * [3H/2,W] uint8: the Y plane [H,W], then U [H/2,W/2], then V [H/2,W/2] -- cv2's I420 layout.  The conversions are OpenCV's
 * cv2.cvtColor COLOR_YUV2RGB_I420 / COLOR_RGB2YUV_I420, bit for bit: the BT.601 limited-range matrix (Y in [16, 235], U / V in
 * [16, 240] nominally; bytes outside are saturated, not refused) in 20-bit fixed point, h = 1 << 19, arithmetic >> 20, sat to
 * [0, 255]:
 *   YUV -> RGB: Y' = max(0, y - 16) 1220542, d = u - 128, e = v - 128;  R = sat((Y' + h + 1673527 e) >> 20),
 *               G = sat((Y' + h - 852492 e - 409993 d) >> 20),  B = sat((Y' + h + 2116026 d) >> 20)
 *   RGB -> YUV: Y = sat((269484 R + 528482 G + 102760 B + h + (16 << 20)) >> 20) for every pixel;
 *               U = sat((-155188 r - 305135 g + 460324 b + h + (128 << 20)) >> 20),
 *               V = sat((460324 r - 385875 g - 74448 b + h + (128 << 20)) >> 20) from the top-left pixel (r, g, b) of each 2 x 2
 *               block only (no averaging).
 * Chroma is nearest-neighbour in both directions: each (u, v) serves its 2 x 2 block, whatever chroma siting a container tags
 * (Y4M's C420jpeg / C420mpeg2 / C420paldv are all read the same way).  Sources tagged BT.709 (most HD video) are decoded with
 * the BT.601 matrix as OpenCV does, which gives a slightly different L than an exact BT.709 decode; an encoder should tag the
 * output BT.601 limited range (ffmpeg: -colorspace bt470bg -color_range tv). */

/* dev_yuv [B,3H/2,W] (I420) -> dev_rgb [B,H,W,3] (COLOR_YUV2RGB_I420); one launch.  DVC_ERR_SHAPE for an odd or < 2 H or W. */
int dvc_i420_to_rgb8(dvc_ctx* ctx, const unsigned char* dev_yuv, int B, int H, int W, unsigned char* dev_rgb, void* stream);
/* dev_rgb [B,H,W,3] -> dev_yuv [B,3H/2,W] (COLOR_RGB2YUV_I420); one launch.  DVC_ERR_SHAPE for an odd or < 2 H or W. */
int dvc_rgb8_to_i420(dvc_ctx* ctx, const unsigned char* dev_rgb, int B, int H, int W, unsigned char* dev_yuv, void* stream);
/* The video calls for I420 sources: frames[s] is clip s's [F,3Hs_s/2,Ws_s] uint8, host-pinned or device memory; geom holds the
 * geometry of the luma plane (Hs_s, Ws_s even); K, the rows, the recurrence, first_last_lab and last_lab_out are as in
 * dvc_colorize_videos_exemplars_rgb8, and exemplars stay colour images (dvc_set_exemplars).
 *   out_i420 == 0: out[s] receives clip s's sRGB frames [K[s],F,h,w,3];
 *   out_i420 == 1: out[s] receives them as I420 frames [K[s],F,3h/2,w];
 * (h, w) the window (Ho, Wo), or the footprint (dvc_source_footprint) when source_resolution is set.
 * Contract: with sRGB output every output byte and last_lab_out equal what dvc_colorize_videos_exemplars_rgb8 (its rows split
 * by clip) or dvc_colorize_videos_source_rgb8 returns for the frames converted by dvc_i420_to_rgb8; with I420 output each frame
 * is dvc_rgb8_to_i420 of that sRGB frame.  1.5 bytes per pixel go up (and down with out_i420).  Launches per frame step: the
 * sRGB call's plus S (one conversion per clip on the ingest stream), plus, with out_i420, one per output size (the window, or
 * each footprint size) on the post-processing stream.  Device memory does not depend on F.  Refuses what the sRGB calls
 * refuse, plus a null out / out[s] or out_i420 outside {0, 1} (DVC_ERR_ARG), an odd Hs or Ws, and with out_i420 a footprint of
 * odd height or width, which CenterPad's crop can give (DVC_ERR_SHAPE), before any launch.  Synchronises `stream` before
 * returning. */
int dvc_colorize_videos_i420(dvc_ctx* ctx, int S, const int* K, const unsigned char* const* frames, int F, const int* geom, int Ho,
                             int Wo, float temperature, const float* first_last_lab, int wls, float wls_lambda, float wls_sigma,
                             int source_resolution, int out_i420, unsigned char* const* out, float* last_lab_out, void* stream);

/* ---- pre / post-processing around the nets (SURVEY.md §8f row 1) ------------------------------ */

/* F.interpolate(x, scale_factor=0.5, mode="bilinear") -- test.py:58,71.  dev_src [planes,H,W] (H, W even) ->
 * dev_dst [planes,H/2,W/2]; planes = B*C of a contiguous NCHW tensor.  dev_src must be 8-byte aligned (the kernel loads
 * pairs of floats; any cudaMalloc / torch allocation is, a view at an odd float offset is not): DVC_ERR_ARG otherwise. */
int dvc_resize_half(dvc_ctx* ctx, const float* dev_src, int planes, int H, int W, float* dev_dst, void* stream);
/* F.interpolate(x, scale_factor=2, mode="bilinear") * scale -- test.py:100-102 (scale = 1.25 there).
 * dev_src [planes,h,w] -> dev_dst [planes,2h,2w]. */
int dvc_upsample2_scaled(dvc_ctx* ctx, const float* dev_src, int planes, int h, int w, float scale, float* dev_dst,
                         void* stream);

/* Output colour conversion of test.py:116-119 = utils/util.py:134-151 (batch_lab2rgb_transpose_mc for one image):
 * Lab = (l + 50, ab) -> skimage.color.lab2rgb (float64: D65 / 2-degree white point, z < 0 -> 0, the 0.2068966 cube
 * threshold, rgb_from_xyz = inv(xyz_from_rgb), sRGB gamma) -> clip [0,1] -> * 255 -> truncation to uint8.
 * dev_l [B,1,H,W] (centred L), dev_ab [B,2,H,W] -> dev_rgb [B,H,W,3] uint8 (the layout cv2 / PIL write). */
int dvc_lab_to_rgb8(dvc_ctx* ctx, const float* dev_l, const float* dev_ab, int B, int H, int W, unsigned char* dev_rgb,
                    void* stream);

/* Ingest colour conversion of test.py:44-45 = RGB2Lab + ToTensor + Normalize (utils/util_distortion.py:18-23,85-100):
 * skimage.color.rgb2lab in float64 (uint8 / 255, inverse sRGB gamma, xyz_from_rgb, D65 / 2-degree white point,
 * 0.008856 cube-root threshold), cast to float32, then L - 50.  dev_rgb [B,H,W,3] uint8 -> dev_lab [B,3,H,W]. */
int dvc_rgb8_to_lab(dvc_ctx* ctx, const unsigned char* dev_rgb, int B, int H, int W, float* dev_lab, void* stream);

/* ContextualLoss_forward.forward(X_features, Y_features, h, feature_centering) (models/ContextualLoss.py:82-126; the default
 * "forward" matching direction of train.py:79), VALUE ONLY -- no backward pass, so it serves evaluation, not training.
 * dev_X [B,C,NX], dev_Y [B,C,NY] (the reference's [B,C,h,w] feature maps, positions flattened), C a multiple of 64;
 * dev_loss [B] = -log(mean_i max_j A_ij).  Runs K7 twice: row maxima, then the online softmax with the per-row temperature
 * h * (1 - max_j f_ij + 1e-5).  Needs a tensor-core correlation mode. */
int dvc_contextual_loss_forward(dvc_ctx* ctx, const float* dev_X, const float* dev_Y, int B, int C, int NX, int NY, float h,
                                int feature_centering, float* dev_loss, void* stream);

/* The "WLS filter" of test.py:105-112: cv2.ximgproc.createFastGlobalSmootherFilter(guide, lambda, sigma_color,
 * lambda_attenuation = 0.25, num_iter = 3).filter(plane) for `planes` fp32 planes [planes,H,W] sharing one single-channel uint8
 * guide [H,W] (Min et al., Fast Global Image Smoothing Based on Weighted Least Squares, TIP 2014: per iteration a horizontal
 * and a vertical sweep of tridiagonal solves (I + lambda_n L) u = f, weights exp(-|dg| / sigma_color), lambda_{n+1} =
 * lambda_n * lambda_attenuation).  dev_dst may equal dev_src.  test.py uses lambda = 500, sigma_color = 4. */
int dvc_fgs_filter(dvc_ctx* ctx, const unsigned char* dev_guide, const float* dev_src, int planes, int H, int W, float lambda,
                   float sigma_color, float lambda_attenuation, int num_iter, float* dev_dst, void* stream);
/* The guide of test.py:106: uint8(uncenter_l(L) * 255 / 100) from the centred luminance plane dev_l [H,W]. */
int dvc_l_to_guide8(dvc_ctx* ctx, const float* dev_l, int H, int W, unsigned char* dev_guide, void* stream);

/* The resize inside CenterPad (utils/util_distortion.py:217-258) and the crop / pad around it:
 * skimage.transform.resize(I, (Hr, Wr), mode="reflect", preserve_range=True, clip=False, anti_aliasing=True) of the uint8
 * image dev_src [Hs,Ws,3] -- float64 Gaussian pre-filter with sigma = max(0, (in/out - 1)/2) per axis (scipy.ndimage
 * gaussian_filter, mode "mirror", truncate 4) then bilinear scipy.ndimage.zoom(order=1, mode="mirror", grid_mode=True) --
 * truncated to uint8; dev_dst [Ho,Wo,3] receives resized[y + oy, x + ox] where that exists and 0 elsewhere (CenterPad's
 * centred crop and torchvision CenterCrop's zero pad; the geometry is computed by the caller, dvc/prepost.py). */
int dvc_resize_antialias_crop_rgb8(dvc_ctx* ctx, const unsigned char* dev_src, int Hs, int Ws, int Hr, int Wr, int oy, int ox,
                                   unsigned char* dev_dst, int Ho, int Wo, void* stream);

/* ---- multi-GPU: exemplar operands travel once per clip (SURVEY.md §8e) ----------------------- */

/* ---- single-frame scaling: query-row-sharded correlation with a fused all-gather (SURVEY.md §8e, BASELINE config 4) --
 * Every row of NonlocalNet.py:477-498 is independent, so G GPUs can each take N/G query rows of one frame against the
 * full exemplar side.  Instead of an NCCL all-gather after the kernel, the kernel that finalises a result row stores it
 * into the full-size result buffer of EVERY GPU through peer-mapped pointers (NVLink stores).  The buffers are plain
 * cudaMalloc allocations shared between the one-process-per-GPU ranks with CUDA IPC. */

/* Allocate `bytes` of device memory and return its IPC handle (64 bytes, cudaIpcMemHandle_t) for the other ranks. */
int dvc_peer_buffer_create(dvc_ctx* ctx, int64_t bytes, void** dev_ptr, unsigned char* handle64);
/* Map another rank's buffer (handle from its dvc_peer_buffer_create) into this process; enables peer access. */
int dvc_peer_buffer_open(dvc_ctx* ctx, const unsigned char* handle64, void** dev_ptr);
int dvc_peer_buffer_close(dvc_ctx* ctx, void* opened_ptr);
int dvc_peer_buffer_destroy(dvc_ctx* ctx, void* created_ptr);
/* Until cleared with n = 0, dvc_corr_softmax_warp (B = 1) additionally stores row r of its result as global row
 * row0 + r into y4[g] ([N_total][4] floats: L, a, b, 0) and sim[g] ([N_total]) for g < n <= 8. */
int dvc_corr_set_peer_outputs(dvc_ctx* ctx, int n, float* const* y4, float* const* sim, int64_t row0);

/* Size in floats of the packed exemplar operands (phi_hat planes + pooled Lab) for an HxW exemplar. */
int64_t dvc_exemplar_pack_size(const dvc_ctx* ctx, int H, int W);
/* Pack the cached exemplar operands into / install them from a flat device buffer, so that the
 * caller can move them with ncclBroadcast (torch.distributed.broadcast) over NVLink. */
int dvc_exemplar_export(dvc_ctx* ctx, float* dev_buf, int64_t n_floats, void* stream);
int dvc_exemplar_import(dvc_ctx* ctx, const float* dev_buf, int64_t n_floats, int H, int W, void* stream);

/* ---- introspection -------------------------------------------------------------------------- */

/* Number of kernels this library launched since the last call with reset != 0. */
int64_t dvc_launch_count(dvc_ctx* ctx, int reset);
/* CUDA-event timing of the correlation kernel: mean milliseconds over the launches recorded since
 * the last reset (0 if none).  Recording is enabled with dvc_profile_corr(ctx, 1). */
int dvc_profile_corr(dvc_ctx* ctx, int enable);
double dvc_corr_mean_ms(dvc_ctx* ctx, int reset);
/* Same for the tensor-core convolution launches: dvc_conv_profile sums the CUDA-event durations (ms) and the
 * algorithmic FLOPs of the recorded launches of one kernel variant (64 / 128 / 256 = pixel-major channel tile,
 * 1 = channel-major kernel, 0 = all) and returns the number of launches. */
int dvc_profile_conv(dvc_ctx* ctx, int enable);
int dvc_conv_profile(dvc_ctx* ctx, int variant, int reset, double* total_ms, double* total_flops);

/* Debug / test hooks (not part of the drop-in surface).
 *   dvc_debug_set_flag: "two_level" (default 1) selects per-tap two-level fp32 accumulation in the
 *   CUDA-core convolution (shorter rounding chain; 0 = plain sequential accumulation, faster).  "keep_stages" (default 0)
 *   gives WarpNet's residual blocks and projection buffers of their own (<tag>.res<i>.raw1 / .mid / .raw2 / .out,
 *   <tag>.proj_raw) instead of reusing two, so every stage can be read after the call; results are bit-identical.
 *   dvc_debug_get_buffer: device pointer / size of a named internal workspace (padded NHWC activations
 *   carry their [B,H,W,C,P] signature in sig5) so tests can check intermediate stages.  "corr.screen_cells" is the
 *   screened T -> 0 correlation's 4 maxima (float bits): query-side ||dropped||, ||hi||, then reference-side. */
int dvc_debug_set_flag(dvc_ctx* ctx, const char* name, int value);
int dvc_debug_get_buffer(dvc_ctx* ctx, const char* name, void** dev_ptr, int64_t* bytes, int* sig5);
/*   dvc_debug_conv2d: ONE convolution layer (the weights `name` of network `net`, already set with dvc_set_weight) on a
 *   device NCHW input, through exactly the engine / operand format / epilogue the layer programs would use under the
 *   current dvc_set_math and debug flags ("tc_force_bn" = 64 / 128 / 256 pins the channel tile) -- the per-layer parity
 *   tests compare it with an fp64 F.conv2d (nn.Conv2d at NonlocalNet.py:235-255,364-423, ColorVidNet.py:96-143).
 *   pad_mode 0 = zero padding, 1 = ReflectionPad2d; act 0 none / 1 ReLU / 2 LeakyReLU(slope); in_bound >= max |x|
 *   (fixes the exact power-of-two scale of the fp16 operand planes), or in_bound < 0 for the first layers (Cin <= 8, no
 *   tensor-core weights): max |x| is measured on the device, as the VGG and ColorVidNet layer programs do; out_planes = 1
 *   stores the result as fp16 hi/lo planes with the device-derived exponent and reads it back (the first layers need
 *   in_bound < 0 for that); upconv = 1: Upsample(2, nearest) + Conv2d(3x3) as four
 *   phase convolutions (y is [B][Cout][2H][2W]); fuse_tail = 1: conv10_2 + LeakyReLU + conv10_ab + tanh*128 (y is
 *   [B][2][H][W]); add: optional device NCHW addend of the output's shape; stats_out: optional device [B][Cout][2]
 *   doubles receiving (sum, sum of squares) over positions. */
int dvc_debug_conv2d(dvc_ctx* ctx, int net, const char* name, const float* dev_x, int B, int H, int W, int dil, int stride,
                     int act, float slope, int pad_mode, int upconv, int fuse_tail, float in_bound, int out_planes,
                     const float* dev_add, float* dev_y, double* dev_stats_out, void* stream);
/*   dvc_debug_resize_taps: host only, no context and no device.  The normalised Gaussian taps that
 *   dvc_resize_antialias_crop_rgb8 and the video ingest give an axis resized from in_len to out_len pixels
 *   (scipy.ndimage._gaussian_kernel1d(sigma = (in_len / out_len - 1) / 2, 0, radius = int(4 sigma + 0.5))): *radius, and the
 *   2 * radius + 1 taps when `capacity` holds them (DVC_ERR_SHAPE when it does not; *radius is set either way).  An axis that
 *   is not down-scaled has no filter: radius 0 and no taps. */
int dvc_debug_resize_taps(int in_len, int out_len, double* taps, int capacity, int* radius);

#ifdef __cplusplus
}
#endif
#endif /* DVC_H_ */
