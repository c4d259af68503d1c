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

/* ---- F.interpolate(scale_factor=2, mode="trilinear", align_corners=False) (decoder.py:105-106), fwd + adjoint */
int b200unet_upsample2x_fwd(const b200unet_tensor* x, const b200unet_tensor* y, double* stats, int stats_ld,
                            void* stream);
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

/* ---- Dice criterion (monai.losses.DiceLoss as configured by script_utils.py:61-77).
 * flags: bit0 sigmoid, bit1 squared_pred, bit2 jaccard, bit3 batch, bit4 exclude background, bit5 reduction=sum,
 * bit6 `target` points to fp32 values (soft labels) instead of uint8.
 * sums: [N][C][3] doubles (I, P, T) written by fwd and consumed by bwd. */
int b200unet_dice_fwd(const float* logits, const void* target, int n, int c, int64_t spatial, int flags,
                      float smooth_nr, float smooth_dr, double* sums, float* loss, void* stream);
int b200unet_dice_bwd(const float* logits, const void* target, int n, int c, int64_t spatial, int flags,
                      float smooth_nr, float smooth_dr, const double* sums, const float* grad_out, float* dlogits,
                      void* stream);

/* ---- Dice + cross-entropy criterion (monai.losses.DiceCELoss): loss = lambda_dice * Dice(act(x), t) + lambda_ce * CE(x, t).
 * Dice is the formula above on p = act(x); include_background = 0 drops channel 0 after the activation.  CE is on the raw
 * logits: -sum_c t_c log_softmax(x)_c for c > 1 (a label map is its one-hot row), BCEWithLogits(x, t) for c == 1; mean
 * divides by n * spatial.  With c == 1 softmax is ignored and a uint8 label map is the target itself (int64: E_UNSUPPORTED).
 * A label outside [0, c) is an all-zero target row.  logits NCDHW fp32, 1 <= c <= 128.
 * scratch: b200unet_dice_ce_scratch_bytes() bytes (0 = the options or shape are rejected), written by fwd and read by bwd.
 * It starts with sums [n][c][3] fp64 (I, P, T) and ce [n] fp64 (the summed CE terms of each sample).  No floating-point
 * atomics: the loss and dlogits are bit-identical run to run. */
typedef struct b200unet_dice_ce_desc {
  int32_t act;                  /* 0 identity, 1 sigmoid, 2 softmax over channels */
  int32_t target_kind;          /* 0 uint8 label map [n][1][spatial], 1 int64 label map, 2 uint8 [n][c][spatial], 3 fp32 [n][c][spatial] */
  int32_t include_background, squared_pred, jaccard, batch;
  int32_t reduction;            /* 0 mean, 1 sum */
  float smooth_nr, smooth_dr, lambda_dice, lambda_ce;
} b200unet_dice_ce_desc;
size_t b200unet_dice_ce_scratch_bytes(const b200unet_dice_ce_desc* desc, int n, int c, int64_t spatial);
int b200unet_dice_ce_fwd(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c,
                         int64_t spatial, void* scratch, float* loss, void* stream);
int b200unet_dice_ce_bwd(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c,
                         int64_t spatial, const void* scratch, const float* grad_out, float* dlogits, void* stream);

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
                                 1,2,2,..., transposed-conv upsampling kernel = stride = 2, InstanceNorm(affine) + LeakyReLU */
  int32_t filters[8];         /* arch 1: channels per level (multiples of 8) */
  float act_slope;            /* arch 1: negative slope of the LeakyReLU (0.01) */
  int32_t deterministic;      /* 1 = weight gradients without floating-point atomics: the split-K CTAs write per-split partial
                                 sums, a second kernel adds them in a fixed order (bit-identical gradients run to run) */
  int32_t inference_only;     /* 1 = forward-only plan (volumetric.py:131-150 runs under no_grad): no backward schedule, no
                                 backward buffers, forward temporaries are recycled -> a much smaller workspace */
  int32_t input_grad;         /* 1 = the plan can also produce d(loss)/d(x) (b200unet_plan_input_grad): saliency maps, adversarial
                                 training, cascades whose input comes from a differentiable stage.  Costs the forward only the data-
                                 gradient weight packs of the first block's convolutions.  Rejected with inference_only = 1. */
} b200unet_net_desc;

typedef struct b200unet_plan b200unet_plan;

int b200unet_plan_create(const b200unet_net_desc* desc, b200unet_plan** out);
void b200unet_plan_destroy(b200unet_plan* plan);
/* number of parameter tensors, in reference state_dict order (SURVEY.md appendix B) */
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
/* The same backward in two calls, so that a data-parallel caller can exchange the gradients that are already final while the
 * rest of the backward runs (the reference's DataParallel reduces every gradient after the whole backward:
 * unet3d/models/build.py:18-20).  backward_parts: 2 when the schedule has a split point (part 0 = head, decoder, deepest
 * encoder level(s): most of the parameters; part 1 = the shallow encoder levels), 1 otherwise, 0 for an inference_only plan.
 * param_backward_part(i): the part after which grads[i] is final.  backward_part(0) followed by backward_part(1) on the same
 * stream writes exactly what b200unet_plan_backward writes; both calls take the same pointers. */
int b200unet_plan_backward_parts(const b200unet_plan* plan);
int b200unet_plan_param_backward_part(const b200unet_plan* plan, int i);
int b200unet_plan_backward_part(b200unet_plan* plan, int part, const float* dlogits, const float* const* params, float* const* grads,
                                void* workspace, void* stream);
/* input gradient of a plan created with input_grad = 1: dx = d(loss)/d(x), NCDHW fp32 [N][n_features][D][H][W], overwritten.
 * Runs after b200unet_plan_backward (or after backward_part(1)) on the same stream and workspace, before the next forward: it reads
 * what that backward left in the workspace (the gradients reaching the first block, the packed input, the first norm's
 * coefficients).  UNet3D: GroupNorm(+ReLU) backward of encoder.layers.0.blocks.0.conv1.norm1 + the data gradient of the block's
 * 1x1x1 `sample` branch or its identity (myronenko.py:34-58); DynUNet: the data gradient of input_block.conv1.  The parameter
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
