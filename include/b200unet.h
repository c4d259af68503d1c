/* libb200unet -- C ABI of the H100-native (sm_90a) 3D U-Net forward/backward hot path.
 *
 * The reference (ellisdg/3DUnetCNN) has no FFI: its extension seam is the Python name lookup
 * unet3d/models/build.py:9-13 (fetch_model_by_name) and unet3d/scripts/script_utils.py:61-77 (load_criterion).
 * This header is the boundary a maintainer binds (ctypes stub: INTEGRATION.md); each entry point names the
 * reference arithmetic it replaces.  All paths below are relative to the reference repository root.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (PyTorch tensors); the library never frees or keeps
 *     caller memory beyond a call, except the opaque plan object created/destroyed explicitly;
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*); no call synchronises the device;
 *   - return value: 0 = ok, <0 = error (b200unet_last_error() gives a thread-local message); there is NO CPU fallback;
 *   - activations are NDHWC bf16 "views": value = hi (+ lo when lo != NULL, the split-precision parity mode),
 *     `c` visible channels out of a buffer with channel pitch `ld` (both multiples of 8);
 *   - model inputs/outputs at the reference-facing boundary are NCDHW fp32, targets uint8 (as the reference's
 *     loaders produce them: unet3d/datasets/segmentation.py:97-122, unet3d/transforms/one_hot.py:10).
 */
#ifndef B200UNET_H_
#define B200UNET_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200UNET_OK 0
#define B200UNET_E_INVALID (-1)
#define B200UNET_E_UNSUPPORTED (-2)
#define B200UNET_E_CUDA (-3)
#define B200UNET_E_DRIVER (-4)

typedef struct b200unet_tensor {
  void* hi;           /* bf16 NDHWC data */
  void* lo;           /* bf16 residual part (value = hi + lo) or NULL */
  int32_t n, d, h, w; /* logical extents */
  int32_t c;          /* visible channels */
  int32_t ld;         /* channel pitch of the underlying buffer, in elements */
} b200unet_tensor;

int b200unet_version(void);
const char* b200unet_last_error(void);

/* ---- layout converters at the NCDHW fp32 boundary (model input: unet3d/train/training_utils.py:109) */
int b200unet_ncdhw_to_ndhwc(const float* x, int c_real, const b200unet_tensor* out, void* stream);
int b200unet_ndhwc_to_ncdhw(const b200unet_tensor* in, int c_real, float* y, void* stream);

/* ---- weight packing.  torch Conv3d weight [Co][Ci][k^3] fp32 (resnet.py:12-22) -> bf16 GEMM operand.
 *   mode 0: [T][Cop][Cip]  forward;  mode 1: [T][Cip][Cop] taps flipped (data gradient);
 *   mode 2: ConvTranspose3d weight [Ci][Co][k^3] (decoder.py:101-102) -> [T][Cop][Cip] flipped;
 *   mode 3: the same weight -> [T][Cip][Cop] unflipped (its data gradient);  mode 4: -> [T][Cop][Cip] unflipped
 *   (forward of a kernel = stride transposed convolution, MONAI UnetUpBlock).
 *   Both entry points: cop and cip multiples of 8 and 1 <= taps <= 27, else B200UNET_E_UNSUPPORTED. */
int b200unet_pack_weights(const float* w, int co, int ci, int cop, int cip, int taps, int mode, void* hi, void* lo,
                          void* stream);
/* fp32 [T][Cip][Cop] accumulator -> torch gradient layout (mode 0: [Co][Ci][T]; mode 2: [Ci][Co][T] flipped) */
int b200unet_unpack_wgrad(const float* g, int co, int ci, int cop, int cip, int taps, int mode, float* out,
                          void* stream);

/* ---- convolution forward / data gradient: nn.Conv3d k{1,3} s{1,2} p=k/2, bias-free (resnet.py:12-22),
 * autograd's bwd-data when called with mode-1 packed weights.  Implicit GEMM on wgmma tensor cores. */
typedef struct b200unet_conv_desc {
  b200unet_tensor x[2];    /* A operands; x[1] only when nsrc == 2 (fused 1x1x1 `sample`, myronenko.py:42-45,53-54) */
  const void* w_hi[2];     /* packed weights per source */
  const void* w_lo[2];
  int32_t ksz[2];          /* 1 or 3 */
  int32_t stride[2];       /* 1 or 2 */
  int32_t cip[2];          /* packed K extent */
  int32_t nsrc;
  int32_t cop;             /* packed weight rows */
  b200unet_tensor out;
  const b200unet_tensor* res;   /* optional residual: `x += identity` (myronenko.py:56) */
  const float* scale;           /* optional [N][C] Dropout3d channel scale (myronenko.py:78-79) */
  double* stats;                /* optional [N][stats_ld][2] (sum, sumsq) for the next GroupNorm */
  int32_t stats_ld;
  int32_t mode;                 /* 0 plain epilogue; 1 GroupNorm+ReLU backward epilogue */
  const b200unet_tensor* gn_x;  /* mode 1: raw input of the norm */
  const float* coef;            /* mode 1: [N][coef_ld][4] from b200unet_gn_apply */
  int32_t coef_ld;
  float slope;                  /* 0 = ReLU (myronenko.py:14), 0.01 = LeakyReLU (DynUNet blocks) */
  double* bstats;               /* mode 1: [N][coef_ld][2] += (sum dz, sum dz*xhat) */
  int32_t cls_mode;             /* 1: data gradient of a k3 s2 p1 convolution (encoder downsampling, myronenko.py:103-105) without
                                   zero insertion: x[0] = dY at half the extent of `out`, weights = the mode-1 pack; plain epilogue */
} b200unet_conv_desc;
int b200unet_conv3d(const b200unet_conv_desc* desc, void* stream);

/* ---- convolution weight gradient (autograd bwd-filter of the same nn.Conv3d): dw fp32 [T][Cip][Cop] += ... */
int b200unet_conv3d_wgrad(const b200unet_tensor* a, const b200unet_tensor* dy, int ksz, int stride, int cip, int cop,
                          float* dw, void* stream);

/* ---- GroupNorm(G, C, eps, affine) + ReLU / LeakyReLU (myronenko.py:17-31): forward and backward, each in one launch.
 * `c` real channels (the length of gamma / beta; NULL gamma = 1, NULL beta = 0) in `groups` groups, out of the x->c channels
 * of the view; x->c is also the channel pitch of stats, coef and bstats.  x->c <= 1024, else B200UNET_E_UNSUPPORTED.
 * The spatial extent is d*h*w of x.  gn_bwd_finalize takes the pitch (c_ld), batch and spatial extent explicitly.
 *   gn_apply:        stats [n][x->c][2] fp64 (sum, sumsq) of each real channel -> coef [n][x->c][4] (A, B, mu, rstd), written
 *                    for the backward (zeros on padded channels), and y = act(A x + B) with act(z) = z > 0 ? z : slope * z
 *   gn_bwd:          bstats [n][x->c][2] fp64 (sum dz, sum dz * xhat) of dz = dL/d(norm output), already masked by act'
 *                    (b200unet_conv3d mode 1, b200unet_act_bwd) -> dx = dL/dx (+ add1) (+ add2); writes dgamma, dbeta
 *                    (either may be NULL)
 *   gn_bwd_finalize: the same without dx: coef2 [n][c_ld][2] = (E, F) of dx = A dz + E x + F, dgamma and dbeta */
int b200unet_gn_apply(const b200unet_tensor* x, const b200unet_tensor* y, const double* stats, const float* gamma,
                      const float* beta, int c, int groups, float eps, float slope, float* coef, void* stream);
int b200unet_gn_bwd(const b200unet_tensor* dz, const b200unet_tensor* x, const float* coef, const double* bstats,
                    const float* gamma, int c, int groups, float* dgamma, float* dbeta, const b200unet_tensor* add1,
                    const b200unet_tensor* add2, const b200unet_tensor* dx, void* stream);
int b200unet_gn_bwd_finalize(const double* bstats, const float* coef, const float* gamma, int n, int c, int c_ld,
                             int groups, int64_t spatial, float* coef2, float* dgamma, float* dbeta, void* stream);

/* ---- post-activation blocks (conv -> norm -> act: MONAI UnetBasicBlock): gradient through the activation of
 * a = act(A c + B):  dz = (g1 [+ g2]) * act'(A c + B),  bstats[n][ch] += (sum dz, sum dz * xhat)  -> b200unet_gn_bwd */
int b200unet_act_bwd(const b200unet_tensor* g1, const b200unet_tensor* g2, const b200unet_tensor* c, const float* coef, float slope,
                     const b200unet_tensor* dz, double* bstats, int bstats_ld, void* stream);

/* ---- MONAI UNet's learnable PReLU (nn.PReLU(num_parameters=1)) after an instance norm, the slope read from the DEVICE fp32
 * scalar `slope` (the parameter itself, so a captured CUDA graph sees every optimizer step's value).
 *   prelu_apply:   gn_apply with act(z) = z > 0 ? z : slope[0] * z, then y = act(z) + add (add: y's shape or NULL; MONAI's
 *                  ResidualUnit output conv(x) + residual(x), the addend read as hi + lo and the sum stored as y's hi [+ lo]).
 *   prelu_bwd:     act_bwd with the same slope; also dslope[0] = sum over z <= 0 of z * (g1 [+ g2]) (written), z = A c + B the
 *                  normalised, affine-applied pre-activation, from per-block partial sums added in a fixed order: bit-identical run
 *                  to run.  scratch: prelu_bwd_scratch_bytes(c).  gsum (optional, c's shape): gsum = g1 [+ g2], the gradient
 *                  a residual branch takes as well. */
int b200unet_prelu_apply(const b200unet_tensor* x, const b200unet_tensor* y, const double* stats, const float* gamma,
                         const float* beta, int c, int groups, float eps, const float* slope, const b200unet_tensor* add, float* coef,
                         void* stream);
size_t b200unet_prelu_bwd_scratch_bytes(const b200unet_tensor* c);
int b200unet_prelu_bwd(const b200unet_tensor* g1, const b200unet_tensor* g2, const b200unet_tensor* c, const float* coef,
                       const float* slope, const b200unet_tensor* dz, double* bstats, int bstats_ld, const b200unet_tensor* gsum,
                       float* dslope, float* scratch, void* stream);

/* ---- logits of a network whose last layer is a convolution (MONAI UNet): logits NCDHW fp32 [n][c_real][d][h][w] =
 * in + bias (+ add) over the first c_real channels of the padded conv result `in` (read as hi + lo); bias DEVICE fp32 [c_real]
 * or NULL; add (in's shape) or NULL: the top residual unit's identity branch, logits = conv(y) + bias + y.  The matching
 * backward pack of dlogits into the padded NDHWC layout is b200unet_ncdhw_to_ndhwc. */
int b200unet_logits_unpack(const b200unet_tensor* in, const b200unet_tensor* add, const float* bias, int c_real, float* logits,
                           void* stream);

/* ---- F.interpolate(scale_factor=2, mode="trilinear", align_corners=False) (decoder.py:105-106), fwd + adjoint.
 * add_fwd: y = upsample(x) + add in one pass (MONAI SegResNet's `up(x) + skip`), add of y's shape (NULL = upsample_fwd); the
 * statistics are those of y.  The gradient of the sum reaches add unchanged and x through upsample2x_bwd. */
int b200unet_upsample2x_fwd(const b200unet_tensor* x, const b200unet_tensor* y, double* stats, int stats_ld,
                            void* stream);
int b200unet_upsample2x_add_fwd(const b200unet_tensor* x, const b200unet_tensor* add, const b200unet_tensor* y, double* stats,
                                int stats_ld, void* stream);
int b200unet_upsample2x_bwd(const b200unet_tensor* dy, const b200unet_tensor* dx, void* stream);
int b200unet_zero_insert(const b200unet_tensor* x, const b200unet_tensor* z, int od, int oh, int ow, void* stream);

/* ---- final 1x1x1 convolution to NCDHW fp32 logits (variational.py:59-60,84-86); act: 0 none 1 sigmoid 2 softmax.
 * n_out is 1..128 and picks the kernels: 1..8 run a SIMT head with fp32 weights (any c that is a multiple of 8); 9..128 run
 * a tensor-core head (bf16 MMAs with fp32 accumulation, c a multiple of 8 up to 64) that rounds the weights -- and in the
 * backward dlogits -- to bf16, or splits them into bf16 hi + lo when x carries a lo plane.  Above 128: E_UNSUPPORTED. */
int b200unet_head_fwd(const b200unet_tensor* x, const float* w, int n_out, int act, float* logits, void* stream);
/* head_bwd reduces dw without floating-point atomics (bit-reproducible for both heads): `scratch` holds one partial per
 * thread block */
size_t b200unet_head_bwd_scratch_bytes(int n_out, int c);
int b200unet_head_bwd(const b200unet_tensor* x, const float* w, int n_out, const float* dlogits,
                      const b200unet_tensor* dx, float* dw, float* scratch, void* stream);

/* ---- Dice criteria (monai.losses.DiceLoss as configured by script_utils.py:61-77, and monai.losses.DiceCELoss).
 * Both take their options in b200unet_dice_ce_desc.  loss = lambda_dice * Dice(act(x), t) + lambda_ce * CE(x, t), where per
 * (n, c) I = sum p*t, P = sum p (or p^2), T = sum t (or t^2) on p = act(x) and f = 1 - (2I + smooth_nr) / (P + T + smooth_dr)
 * [jaccard: denominator 2(P + T - I)]; batch pools I, P, T over n; Dice is the mean (or sum) of f; include_background = 0 drops
 * channel 0 after the activation. */
typedef struct b200unet_dice_ce_desc {
  int32_t act;                  /* 0 identity, 1 sigmoid, 2 softmax over channels */
  int32_t target_kind;          /* 0 uint8 label map [n][1][spatial], 1 int64 label map, 2 uint8 [n][c][spatial], 3 fp32 [n][c][spatial] */
  int32_t include_background, squared_pred, jaccard, batch;
  int32_t reduction;            /* 0 mean, 1 sum */
  float smooth_nr, smooth_dr, lambda_dice, lambda_ce;
  /* Everything below is the dice_ce entry points' alone; zeroed, it is the Dice overlap with the CE term above. */
  int32_t overlap;              /* 0 Dice; 1 Tversky (monai.losses.TverskyLoss): f = 1 - (I + smooth_nr) / (I + tversky_alpha (P - I)
                                   + tversky_beta (T - I) + smooth_dr); 2 generalized Dice (GeneralizedDiceLoss): per sample (once
                                   with batch) f = 1 - (2 sum_c w_c I_c + smooth_nr) / (sum_c w_c (P_c + T_c) + smooth_dr), w_c from
                                   T_c by w_type, an infinite weight replaced by the largest finite one of the sample (of all, with
                                   batch); squared_pred and jaccard 0 for both */
  float tversky_alpha, tversky_beta;
  int32_t w_type;               /* generalized Dice: 0 1/T^2, 1 1/T, 2 uniform */
  int32_t voxel_term;           /* the term lambda_ce scales: 0 CE, 1 focal (monai.losses.FocalLoss) on the channels include_background
                                   keeps; mean divides its total by n * c' * spatial, sum by spatial (MONAI averages over the voxels);
                                   2 distance-weighted (monai.losses.HausdorffDTLoss), (p_c - t_c)^2 hdt_weight on the kept channels
                                   with p = act(x), divided as focal, and by n * spatial for sum with batch; lambda_dice 0 */
  int32_t focal_softmax;        /* 0 sigmoid form, per element (x - x t - logsigmoid(x)) exp(gamma logsigmoid(-x (2t - 1)));
                                   1 softmax form -(1 - exp(ls))^gamma ls t, ls = log_softmax over the kept channels */
  float focal_gamma;            /* >= 0 */
  float focal_alpha;            /* with focal_use_alpha: sigmoid t alpha + (1 - t)(1 - alpha), softmax 1 - alpha on the first kept
                                   channel and alpha on the others */
  int32_t focal_use_alpha;
  const float* class_weight;    /* focal: DEVICE fp32 [c'] per-class factors, NULL = none */
  const float* hdt_weight;      /* distance-weighted: DEVICE fp32 [n][c'][spatial] from b200unet_hausdorff_dt_weight */
} b200unet_dice_ce_desc;

/* DiceLoss: act 0 or 1 (softmax: E_UNSUPPORTED, b200unet_dice_ce_* runs it), target_kind 2 or 3 (label maps: E_UNSUPPORTED),
 * lambda_ce 0 (else E_INVALID), overlap and voxel_term 0 (else E_UNSUPPORTED); any c >= 1.  logits NCDHW fp32.
 * scratch: [n][c][3] fp64 sums (I, P, T) followed by [n][c][2] fp64 backward coefficients, written by fwd and read by bwd.
 * The sums are added with fp64 atomics, so the loss may differ in its last bits from run to run. */
int b200unet_dice_fwd(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c,
                      int64_t spatial, double* scratch, float* loss, void* stream);
int b200unet_dice_bwd(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c,
                      int64_t spatial, const double* scratch, const float* grad_out, float* dlogits, void* stream);

/* DiceCELoss: CE is on the raw logits: -sum_c t_c log_softmax(x)_c for c > 1 (a label map is its one-hot row),
 * BCEWithLogits(x, t) for c == 1; mean divides by n * spatial.  lambda_ce = 0 means the CE (or focal) term is not evaluated, so logits of +-inf give a finite sigmoid Dice
 * loss and gradient; lambda_dice = 0 likewise skips the overlap sums.  The same entry points run TverskyLoss, GeneralizedDiceLoss,
 * FocalLoss and DiceFocalLoss through the descriptor's tail.  With c == 1 softmax is ignored and a uint8 label map is the target itself (int64: E_UNSUPPORTED).
 * A label outside [0, c) is an all-zero target row.  logits NCDHW fp32, 1 <= c <= 128.
 * scratch: b200unet_dice_ce_scratch_bytes() bytes (0 = the options or shape are rejected), written by fwd and read by bwd.
 * It starts with sums [n][c][3] fp64 (I, P, T) and ce [n] fp64 (the summed CE terms of each sample).  No floating-point
 * atomics: the loss and dlogits are bit-identical run to run. */
size_t b200unet_dice_ce_scratch_bytes(const b200unet_dice_ce_desc* desc, int n, int c, int64_t spatial);
int b200unet_dice_ce_fwd(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c,
                         int64_t spatial, void* scratch, float* loss, void* stream);
int b200unet_dice_ce_bwd(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c,
                         int64_t spatial, const void* scratch, const float* grad_out, float* dlogits, void* stream);

/* ---- distance weights of HausdorffDTLoss (monai.losses.HausdorffDTLoss, Karimi & Salcudean 2019), without scipy on the host.
 * For each (n, c) that include_background keeps, the prediction mask act(x) > 0.5 (act, and a softmax over all c channels, as
 * the dice_ce kernels form p) and the target mask t > 0.5 (target_kind as for dice_ce; a label outside [0, c) is no class) each
 * get the field edt(mask) + edt(~mask): per voxel the Euclidean distance, in voxels, to the nearest voxel of the other value,
 * scipy.ndimage.distance_transform_edt's fp64 value rounded to fp32 (bit for bit).  An empty or full mask has the field 0; the
 * rule is applied from device counts, nothing is read back.  weight DEVICE fp32 [n][c'][d*h*w] = pdt^alpha + tdt^alpha, alpha > 0.
 * The desc's act, target_kind and include_background are read; with c == 1 softmax is ignored and a uint8 label map is the
 * target itself.  Extents 1..256 per axis, n * c' <= 4096, c <= 128, else B200UNET_E_UNSUPPORTED.
 *   hausdorff_dt_scratch_bytes: from the shape alone (0 = rejected): 24 bytes per kept (n, c) and voxel. */
size_t b200unet_hausdorff_dt_scratch_bytes(const b200unet_dice_ce_desc* desc, int n, int c, int d, int h, int w);
int b200unet_hausdorff_dt_weight(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c, int d, int h,
                                 int w, float alpha, void* scratch, float* weight, void* stream);

/* ---- sliding-window inference on the device (monai.inferers.SlidingWindowInferer as called by
 * predict/volumetric.py:147-148 and train/training_utils.py:106-107).  `starts`: HOST array [ntiles][4] of
 * (sample, d0, h0, w0), at most 16 tiles per call; volumes and tiles are NCDHW fp32.
 *   gather:    tiles[b] = vol[sample_b, :, d0:d0+rd, h0:h0+rh, w0:w0+rw]
 *   scatter:   out[sample_b, :, window_b] += pred[b] * importance   (tile order, deterministic: no atomics)
 *   count:     cnt[d][h][w] = sum of `importance` over the full scan (separable DEVICE start lists per axis)
 *   normalize: out[nc][v] /= cnt[v] */
int b200unet_tiles_gather(const float* vol, int n, int c, int d, int h, int w, const int32_t* starts, int ntiles, int rd, int rh,
                          int rw, float* tiles, void* stream);
int b200unet_tiles_scatter(const float* pred, int c, const int32_t* starts, int ntiles, int rd, int rh, int rw,
                           const float* importance, float* out, int n, int d, int h, int w, void* stream);
int b200unet_tiles_count(const int32_t* starts_d, int nd, const int32_t* starts_h, int nh, const int32_t* starts_w, int nw, int rd,
                         int rh, int rw, const float* importance, float* cnt, int d, int h, int w, void* stream);
int b200unet_tiles_normalize(float* out, const float* cnt, int nc, int64_t spatial, void* stream);

/* ---- the step before the path: label map -> one-hot uint8 target (utils/one_hot.py:7-37; `values`/`begin` are HOST
 * arrays: channel c is 1 where isclose(round(data), values[k]) for any k in [begin[c], begin[c+1])), and z-score
 * intensity normalisation (monai NormalizeIntensity selected by datasets/segmentation.py:77-87; `groups` = C when
 * channel_wise else 1; stats: [groups][3] doubles of scratch). */
int b200unet_one_hot(const float* data, int n, int64_t spatial, const float* values, const int32_t* begin, int n_channels,
                     int do_round, uint8_t* y, void* stream);
int b200unet_zscore(const float* x, int groups, int64_t spatial, int nonzero, double* stats, float* y, void* stream);
/* ---- the step after the path: activation (0 none, 1 sigmoid, 2 softmax) + threshold -> int16 label map of ONE sample
 * p [L][spatial] (utils/one_hot.py:46-118: label hierarchy, any/sum-then-threshold + argmax).  one_hot and label_map take
 * 1..128 channels; one_hot at most 256 label values in all. */
int b200unet_label_map(const float* p, int n_labels, int64_t spatial, const int32_t* labels, int act, float threshold,
                       int hierarchy, int sum_then_threshold, int16_t* out, void* stream);

/* ---- random augmentation of a training batch (MONAI RandFlipd / RandRotated, NormalizeIntensityd, RandScaleIntensityd /
 * RandShiftIntensityd as datasets/segmentation.py:72-94 chains them), two passes over the image.
 *   scratch_bytes: from the shape alone (0 = rejected: 1..16 image channels, d*h*w < 2^31).  The scratch starts with stats
 *                  [n][c][3] fp64 (sum, sumsq, count) of the resampled image, over the non-zero voxels when nonzero = 1.
 *   resample:      image fp32 [n][c][d][h][w] -> image_out (trilinear), label uint8 [n][l][d][h][w] -> label_out (nearest, round
 *                  half to even; l = 0: no label).  affine: DEVICE fp32 [n][3][4], output index (d, h, w, 1) -> source index.
 *                  padding 0 = border (clamp the source coordinate to [0, size-1]), 1 = zeros; as grid_sample(align_corners=False)
 *                  on index coordinates.  Corners of weight 0 are not read: an axis flip copies every value bit for bit.
 *                  Writes the stats of image_out.
 *   intensity:     in place on the resampled image, after resample with the same scratch: y = ((x - mean) / std) * a + b with
 *                  coef DEVICE fp32 [n][c][2] = (a, b); statistics per (n, c) when channel_wise, else per n; std 0 -> 1;
 *                  normalize = 0: y = x * a + b, and planes with (a, b) = (1, 0) stay untouched; nonzero = 1: zero voxels
 *                  skip the z-score.  Any 4-byte aligned image pointer (16-byte aligned ones with d*h*w a multiple of 4 take
 *                  vector loads).
 * No floating-point atomics: bit-identical run to run. */
size_t b200unet_augment_scratch_bytes(int n, int c, int64_t spatial);
int b200unet_augment_resample(const float* image, const uint8_t* label, int n, int c, int l, int d, int h, int w, const float* affine,
                              int padding, int nonzero, float* image_out, uint8_t* label_out, void* scratch, void* stream);
int b200unet_augment_intensity(float* image, int n, int c, int64_t spatial, int normalize, int nonzero, int channel_wise,
                               const float* coef, void* scratch, void* stream);

/* ---- foreground crop + resize of a training batch of different extents, composed with the augmentation into the one resample
 * above (MONAI CropForegroundD with the reference's percentile_threshold, then ResizeD, as datasets/segmentation.py:55-70 chains
 * them lazily).  samples: DEVICE int64 [n][5] rows (image pointer, label pointer or 0, d, h, w): sample i is fp32
 * [c][d][h][w] and uint8 [l][d][h][w], each fewer than 2^31 voxels per channel.
 *   foreground_scratch_bytes: from (n, c) alone (0 = rejected: 1..16 channels, 1..65535 samples, n * c <= 65535).
 *   foreground_box: crop = 0 takes every whole volume; otherwise the mask is any_c(x_c > thr_c) with thr = 0 (ranks NULL,
 *                  MONAI's default select_fn) or thr_c the linear interpolation, weight gamma DEVICE fp32 [n][c], between
 *                  the order statistics of ranks DEVICE int64 [n][c][2] (np.percentile's two neighbours), written to
 *                  threshold DEVICE fp32 [n][c] (NaN when the channel holds a NaN).  Box per axis [first - margin, last +
 *                  margin + 1), clipped to the volume when allow_smaller; an empty mask takes the whole volume and sets
 *                  empty[i] = 1.  box DEVICE int32 [n][3][2] (start, end).  affine DEVICE fp64 [n][3][4] (index space on the
 *                  (d, h, w) output grid) -> affine_out DEVICE fp32 [n][3][4] onto the sample's own grid:
 *                  box start + s * (A p) + (s - 1) / 2, s = box size / output size.  max_spatial: the largest d*h*w of the
 *                  batch (sizes the grids).  Nothing is read back to the host.
 *   augment_resample_samples: augment_resample onto the (d, h, w) output grid, sample i read from samples[i] at its own extents
 *                  (affine_out above); the output, the scratch and augment_intensity are as for augment_resample. */
size_t b200unet_foreground_scratch_bytes(int n, int c);
int b200unet_foreground_box(const int64_t* samples, int n, int c, int64_t max_spatial, int crop, const int64_t* ranks,
                            const float* gamma, int margin, int allow_smaller, const double* affine, int d, int h, int w,
                            float* affine_out, int32_t* box, int32_t* empty, float* threshold, void* scratch, void* stream);
int b200unet_augment_resample_samples(const int64_t* samples, int n, int c, int l, int d, int h, int w, const float* affine,
                                      int padding, int nonzero, float* image_out, uint8_t* label_out, void* scratch, void* stream);

/* ---- a prediction back onto the grid of its image file (monai.transforms.ResampleToMatch as predict/volumetric.py:135-137,
 * 168-170 calls it): src fp32 [c][sd][sh][sw] -> dst fp32 [c][dd][dh][dw], 1 <= c <= 128, fewer than 2^31 voxels per channel.
 * affine: HOST fp64 row-major 3x4, target index (d, h, w, 1) -> source index (inv(A_src) A_dst with voxel centres on integers),
 * copied by value.  mode 0 = trilinear (fp64 coordinate, fp32 weights), 1 = nearest (round half to even).  Border padding:
 * the source coordinate is clamped to [0, size-1].  Corners of weight 0 are not read: an identity, integer shift, flip or
 * axis permutation copies every value bit for bit. */
int b200unet_resample_to_grid(const float* src, int c, int sd, int sh, int sw, const double affine[12], int mode, float* dst, int dd,
                              int dh, int dw, void* stream);

/* ---- connected components of binary masks (the clean-up after the path: SimpleITK ConnectedComponent + RelabelComponent,
 * MONAI KeepLargestConnectedComponent).  mask uint8 [nvol][d][h][w], nonzero = foreground; each volume is labelled on its own;
 * d*h*w < 2^31.  connectivity in orthogonal hops: 1 = 6 face neighbours, 2 = 18 (+ edges), 3 = 26 (+ corners).
 *   scratch_bytes: from the shape alone (0 = rejected); one buffer serves both calls.
 *   label:         labels int32 [nvol][d][h][w]: 0 background, 1..K_v numbered in raster order of each component's first voxel
 *                  (scipy.ndimage.label); counts int32 [nvol] = K_v.  The component sizes stay in scratch for sort_by_size.
 *   sort_by_size:  in place, after label with the same scratch: renumber by decreasing size, equal sizes in raster order
 *                  (RelabelComponent(sortByObjectSize=True)).  max_count = max_v K_v, read back by the caller.  Consumes the sizes.
 * Exact integers, independent of scheduling. */
size_t b200unet_cc_scratch_bytes(int nvol, int d, int h, int w);
int b200unet_cc_label(const uint8_t* mask, int nvol, int d, int h, int w, int connectivity, int32_t* labels, int32_t* counts,
                      void* scratch, void* stream);
int b200unet_cc_sort_by_size(int32_t* labels, int nvol, int d, int h, int w, int max_count, void* scratch, void* stream);

/* ---- boundary-distance scores of binary segmentations (the scoring after the path: MONAI HausdorffDistanceMetric,
 * SurfaceDistanceMetric, SurfaceDiceMetric on one-hot [b][c][d][h][w] masks, without scipy on the host).  A voxel is foreground
 * iff its value is 1; edges = fg & ~erode(fg) with the 6-neighbour cross, outside the volume = background.  For each of the
 * b x c (item, class) pairs the distances from every edge voxel of one mask to the nearest edge voxel of the other come from an
 * exact Euclidean distance transform, sqrt(((dd s_d)^2 + (dh s_h)^2) + (dw s_w)^2) in fp64 rounded to fp32 as
 * scipy.ndimage.distance_transform_edt computes it (bit for bit with unit spacing).  Extents 1..256 per axis, b x c <= 4096,
 * else B200UNET_E_UNSUPPORTED.
 *   surface_scratch_bytes: from the shape alone (0 = rejected).
 *   surface_distance: spacing DEVICE fp64 [b][3] (d, h, w); q = 0: Hausdorff is the max distance, q in (0, 1]: torch.quantile(d, q)
 *                  on the fp32 distances; hd_dirs / asd_dirs: 1 = pred -> gt only, 2 = both directions (HD: max of the two
 *                  statistics; ASD: mean over both distance sets together, in fp64); nsd: (#{d_pg <= tau} + #{d_gp <= tau}) /
 *                  (n_pg + n_gp) with tau DEVICE fp32 [c].  hd, asd, nsd: DEVICE fp32 [b][c], any of them NULL = not computed.
 *                  Both masks empty: NaN; exactly one empty: HD = ASD = inf, NSD = 0.  Launches do not depend on b x c, nothing is
 *                  read back to the host, no floating-point atomics: bit-identical run to run. */
typedef struct b200unet_surface_mask {
  const void* data;
  int32_t dtype;        /* 0 bool / uint8, 1 fp32 */
  int64_t stride[5];    /* elements, for (b, c, d, h, w) */
} b200unet_surface_mask;
size_t b200unet_surface_scratch_bytes(int b, int c, int d, int h, int w);
int b200unet_surface_distance(const b200unet_surface_mask* pred, const b200unet_surface_mask* gt, int b, int c, int d, int h, int w,
                              const double* spacing, float q, int hd_dirs, int asd_dirs, const float* tau, float* hd, float* asd,
                              float* nsd, void* scratch, void* stream);

/* ---- overlap counts of segmentations (the scoring after the path: MONAI DiceMetric, MeanIoU, ConfusionMatrixMetric), in one
 * pass over the batch.  For every (item, class) pair, counts[b][cls] = (P, G, I): voxels predicted as cls, voxels whose target is
 * cls, voxels that are both.  For binary masks tp = I, fp = P - I, fn = G - I and tn = d*h*w - P - G + I.  An operand is read as:
 *   kind 0 one-hot     [b][c][d][h][w], dtype 0 (bool / uint8) or 2 (fp32): class cls iff the value is nonzero;
 *   kind 1 label map   [b][1][d][h][w], dtype 0 (uint8) or 1 (int64): the class is the value; a value outside [0, c) is no class;
 *   kind 2 threshold   [b][c][d][h][w], dtype 2: class cls iff the value is >= threshold (prediction only);
 *   kind 3 argmax      [b][c][d][h][w], dtype 2: the class is the first channel of the largest value, NaN counting as the
 *                      largest, as torch.argmax (prediction only).
 * Operands are contiguous.  1 <= c <= 128, 1 <= b <= 65535, d*h*w < 2^31, else B200UNET_E_UNSUPPORTED; another kind / dtype pair:
 * B200UNET_E_UNSUPPORTED.  counts: DEVICE int64 [b][c][3], overwritten; exact integers, bit-identical run to run.  Nothing is
 * read back to the host: the call can be captured in a CUDA graph. */
typedef struct b200unet_overlap_operand {
  const void* data;
  int32_t kind;         /* 0 one-hot, 1 label map, 2 threshold, 3 argmax */
  int32_t dtype;        /* 0 bool / uint8, 1 int64, 2 fp32 */
  float threshold;      /* kind 2 */
} b200unet_overlap_operand;
int b200unet_overlap_counts(const b200unet_overlap_operand* pred, const b200unet_overlap_operand* gt, int b, int c, int d, int h,
                            int w, int64_t* counts, void* stream);

/* ---- whole-network plan: UNet3D forward/backward (segmentation/unet.py:7-50, classification/myronenko.py,
 * classification/decoder.py:73-130, autoencoder/variational.py:37-87) as one schedule of the kernels above. */
typedef struct b200unet_net_desc {
  int32_t n_features, n_outputs, base_width;
  int32_t n_levels;
  int32_t encoder_blocks[8];
  int32_t decoder_blocks[8];
  int32_t feature_dilation;
  int32_t norm_groups;
  int32_t use_transposed_convolutions;
  int32_t activation;         /* 0 none, 1 sigmoid, 2 softmax (variational.py:62-68) */
  int32_t split_precision;    /* 0 = bf16 single pass (perf), 1 = hi/lo split, 3 MMAs (parity) */
  int32_t batch, depth, height, width;
  int32_t arch;               /* 0 = the reference's UNet3D (above); 1 = MONAI DynUNet blocks as trained by
                                 examples/brats2020/brats2020_config.json:2-107: n_levels = len(filters), kernel 3, strides
                                 1,2,2,..., transposed-conv upsampling kernel = stride = 2, InstanceNorm(affine) + LeakyReLU;
                                 2 = MONAI SegResNet (GroupNorm pre-activation residual blocks, stride-2 3x3x3 down-sampling,
                                 1x1x1 conv + trilinear x2 + additive skip, GroupNorm + act + biased 1x1x1 head) with
                                 base_width = init_filters (a multiple of 8), n_levels = len(blocks_down), encoder_blocks =
                                 blocks_down, decoder_blocks = blocks_up (n_levels - 1 entries, all >= 1), norm_groups =
                                 num_groups (dividing init_filters); Dropout3d(dropout_prob) on convInit's output through
                                 dropout_scale [N][init_filters].  Rejected with B200UNET_E_UNSUPPORTED: extents not even at
                                 every level above the last, widths above 1024, more than 8 outputs from more than 64 channels */
  int32_t filters[8];         /* arch 1: channels per level (multiples of 8) */
  float act_slope;            /* every architecture: negative slope of the activation after each norm; 0 = the reference
                                 UNet3D's (and SegResNet's default) ReLU, 0.01 = DynUNet's LeakyReLU */
  int32_t deterministic;      /* 1 = weight gradients without floating-point atomics: the split-K CTAs write per-split partial
                                 sums, a second kernel adds them in a fixed order (bit-identical gradients run to run) */
  int32_t inference_only;     /* 1 = forward-only plan (volumetric.py:131-150 runs under no_grad): no backward schedule, no
                                 backward buffers, forward temporaries are recycled -> a much smaller workspace */
  int32_t input_grad;         /* 1 = the plan can also produce d(loss)/d(x) (b200unet_plan_input_grad): saliency maps, adversarial
                                 training, cascades whose input comes from a differentiable stage.  Costs the forward only the data-
                                 gradient weight packs of the first block's convolutions.  Rejected with inference_only = 1. */
  /* arch 3 = MONAI UNet (monai/networks/nets/unet.py): n_levels = len(channels) (2..8), filters = channels (multiples of 8 up
   * to 1024), every stride 2, kernel_size = up_kernel_size = 3, InstanceNorm3d (eps 1e-5) and the activation after every conv
   * but the last; n_features = in_channels 1..16, n_outputs = out_channels 1..16, activation 0.  The fields below are arch 3's
   * alone (zero elsewhere). */
  int32_t num_res_units;      /* 0: Convolution layers; r > 0: ResidualUnit(subunits = r) down layers and up layers followed by a
                                 one-subunit ResidualUnit */
  int32_t act_kind;           /* 0: act_slope (0 ReLU, else LeakyReLU); 1: PReLU with one learnable slope per layer (adn.A.weight) */
  int32_t norm_affine;        /* 1: the instance norms have a weight and a bias (adn.N.weight / .bias) */
  int32_t conv_bias;          /* 1: every convolution has a bias (MONAI's bias=True) */
} b200unet_net_desc;

typedef struct b200unet_plan b200unet_plan;

int b200unet_plan_create(const b200unet_net_desc* desc, b200unet_plan** out);
void b200unet_plan_destroy(b200unet_plan* plan);
/* number of parameter tensors, in reference state_dict order (SURVEY.md appendix B; arch 1, 2 and 3: MONAI's registration order) */
int b200unet_plan_num_params(const b200unet_plan* plan);
/* shape (up to 5 dims, zero padded) and state_dict key of parameter i */
int b200unet_plan_param_info(const b200unet_plan* plan, int i, int64_t shape[5], char* key, int key_cap);
size_t b200unet_plan_workspace_bytes(const b200unet_plan* plan);
/* forward: x NCDHW fp32 -> logits NCDHW fp32.  params: device array-of-pointers (host array of device pointers) to
 * the fp32 parameters.  dropout_scale: [N][C0] per-channel scale or NULL (eval).  save_for_backward: bit 0 states that
 * b200unet_plan_backward will follow (rejected on an inference_only plan, whose workspace keeps no activations); bit 1
 * states that the parameters are unchanged since the previous forward on this workspace (its packed bf16 weights are
 * kept: tiled inference runs many forwards per volume on fixed weights). */
int b200unet_plan_forward(b200unet_plan* plan, const float* x, const float* const* params, const float* dropout_scale,
                          int save_for_backward, void* workspace, float* logits, void* stream);
/* backward: dlogits NCDHW fp32 -> grads[i] (fp32, same shapes as params; overwritten). */
int b200unet_plan_backward(b200unet_plan* plan, const float* dlogits, const float* const* params, float* const* grads,
                           void* workspace, void* stream);
/* input gradient of a plan created with input_grad = 1: dx = d(loss)/d(x), NCDHW fp32 [N][n_features][D][H][W], overwritten.
 * Runs after b200unet_plan_backward on the same stream and workspace, before the next forward: it reads
 * what that backward left in the workspace (the gradients reaching the first block, the packed input, the first norm's
 * coefficients).  UNet3D: GroupNorm(+ReLU) backward of encoder.layers.0.blocks.0.conv1.norm1 + the data gradient of the block's
 * 1x1x1 `sample` branch or its identity (myronenko.py:34-58); DynUNet: the data gradient of input_block.conv1; SegResNet: that of
 * convInit.  The parameter
 * gradients come from the backward alone: this call writes nothing but dx. */
int b200unet_plan_input_grad(b200unet_plan* plan, float* dx, void* workspace, void* stream);
/* number of kernels the last forward / backward / input-gradient call launched (for bench.py's gpu_launches) */
int b200unet_plan_last_launches(const b200unet_plan* plan);

/* per-category accounting for bench.py's roofline (categories: 0 conv fwd, 1 conv dgrad, 2 conv wgrad, 3 norm/act,
 * 4 resample/pack-input, 5 head, 6 weight pack/unpack, 7 other).  algorithmic_macs: conv MACs of ONE forward+backward
 * pass (dgrad excludes the convolutions that read the network input; stride-2 dgrad counted at its true size).
 * profile_begin/end bracket any number of forward/backward calls: every launch is timed with a CUDA-event pair on
 * the launching stream; profile_end synchronises those events and returns summed milliseconds and launch counts. */
int b200unet_plan_algorithmic_macs(const b200unet_plan* plan, double* macs, int ncat);
int b200unet_plan_profile_begin(b200unet_plan* plan, int max_launches);
int b200unet_plan_profile_end(b200unet_plan* plan, double* ms_by_cat, int64_t* launches_by_cat, int ncat);
/* while profiling: write one CSV row per recorded launch (index, category, milliseconds, op label) */
int b200unet_plan_profile_dump(b200unet_plan* plan, const char* path);

#ifdef __cplusplus
}
#endif
#endif /* B200UNET_H_ */
