/* libb200unet diagnostics -- entry points outside the product ABI (include/b200unet.h).
 *
 * They report which kernel a convolution or weight gradient runs on, and launch the operation with the options that only
 * the whole-network plans set otherwise (bias, zeroed boundary, visible extents, deterministic weight-gradient partial sums),
 * so that tests can hold every kernel route to a reference.  The route queries are host-only: they launch nothing, and read
 * the tensors' shapes and which of their pointers are NULL, never the data.  The convolution route asks the runtime for the
 * current device's SM count, which sizes the persistent halo kernel's grid.  Same conventions and
 * status codes as b200unet.h.
 */
#ifndef B200UNET_DIAG_H_
#define B200UNET_DIAG_H_

#include "b200unet.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Options b200unet_conv_desc and b200unet_conv3d_wgrad cannot express.  Every entry point below takes it as NULL = none.
 * Visible extents (d, h, w), 0 = the full extent: voxels at or beyond them read as zero (the masked gradient of a padded
 * ConvTranspose3d output). */
typedef struct b200unet_diag_ext {
  const float* bias;       /* conv, mode 0: per-output-channel bias added after the residual and scale */
  int32_t zero_last;       /* conv, mode 0: output voxels on the high boundary plane, row and column are stored as 0 */
  int32_t x_vis[2][3];     /* conv: visible extents of each source */
  int32_t a_vis[3];        /* weight gradient: of the activation */
  int32_t dy_vis[3];       /* weight gradient and bias gradient: of dy */
  int32_t max_ctas;        /* conv, halo kind on the persistent kernel: > 0 caps its CTAs per N tile (grid[0]), so that small
                              shapes walk several voxel tiles per CTA */
  int32_t tile128;         /* conv, tap kind: != 0 keeps the 128-voxel tile of one consumer warpgroup where the route would take
                              the 256-voxel tile of two (same MMA order per output row: the bf16 output is the same bit for bit) */
} b200unet_diag_ext;

/* kernel kinds of b200unet_conv_route */
#define B200UNET_CONV_TAP 0      /* per-tap streaming tiles */
#define B200UNET_CONV_HALO 1     /* one halo box per K chunk for an 8 x 16 x 1 output tile */
#define B200UNET_CONV_CLASS1 2   /* parity classes: data gradient of a 3x3x3 stride-2 convolution */
#define B200UNET_CONV_CLASS2 3   /* parity classes: ConvTranspose3d with kernel = stride = 2 */
#define B200UNET_CONV_HALO_PAIR 4   /* one halo box for two 8 x 16 x 1 output tiles in consecutive planes, one per consumer
                                       warpgroup; grid[0] counts CTAs, each walking units of two tiles */

typedef struct b200unet_conv_route {
  int32_t kind;
  int32_t bn, kc;                 /* output channels per CTA, input channels per K chunk */
  int32_t kchunks[2];             /* K chunks of each source */
  int32_t npass;                  /* 1 bf16, 3 split precision */
  int32_t cls_pair;               /* class mode in bf16: the two W-parity classes share one store */
  int32_t tw, th, td;             /* output voxel tile of a CTA (class mode: of one parity class) */
  int32_t grid[3];
  int32_t stages, blocks_per_sm, smem_bytes;   /* of the kernel's compile-time configuration */
  int32_t wgs;                    /* consumer warpgroups per CTA: 2 for per-tap tiles of 256 voxels (each warpgroup computes the
                                     half at d0 and d0 + td / 2) and for the two-plane halo kind, 1 otherwise */
} b200unet_conv_route;

/* kernel kinds of b200unet_wgrad_route */
#define B200UNET_WGRAD_SIMT 0    /* 1x1x1 with 8 or 16 input channels, register tiles, atomics only */
#define B200UNET_WGRAD_TAP 1     /* tensor cores, one TMA box per (tap, channel chunk) */
#define B200UNET_WGRAD_HALO 2    /* tensor cores, one halo box per 8 x 16 x 1 voxel tile */

typedef struct b200unet_wgrad_route {
  int32_t kind;
  int32_t ci8;                    /* SIMT: input channels / 8 */
  int32_t cb, bn, qt;             /* input channels per M box, output channels per N tile, M tiles per CTA (per work item) */
  int32_t groups, cotiles, kblocks; /* M-tile groups (groups x cotiles work items), N tiles, voxel tiles */
  int32_t splits;                 /* halo: CTAs per work item; per-tap: the most CTAs sharing one work item (partial slots) */
  int32_t npass;
  int32_t tw, th, td;
  int64_t part_bytes;             /* deterministic mode: splits * taps * cip * cop * 4, the partial-sum buffer it fills */
  int32_t ctas;                   /* tensor-core kinds: CTAs of the launch (per-tap: min(SMs, work items x voxel tiles)) */
} b200unet_wgrad_route;

/* the route b200unet_conv3d / b200unet_diag_conv3d_ex take for this descriptor on the current device (132 SMs without one); an
 * error when they would refuse it */
int b200unet_diag_conv3d_route(const b200unet_conv_desc* desc, const b200unet_diag_ext* ext, b200unet_conv_route* route);
/* the route of b200unet_diag_wgrad_ex (deterministic = a partial buffer is passed) on a device with num_sms SMs */
int b200unet_diag_wgrad_route(const b200unet_tensor* a, const b200unet_tensor* dy, int ksz, int stride, int cip, int cop,
                              const b200unet_diag_ext* ext, int deterministic, int num_sms, b200unet_wgrad_route* route);
/* the partial-buffer bytes the plans allocate for this weight gradient (covers either tiling) */
size_t b200unet_diag_wgrad_partial_bytes(const b200unet_tensor* a, const b200unet_tensor* dy, int ksz, int stride, int cip, int cop,
                                         const b200unet_diag_ext* ext, int num_sms);

int b200unet_diag_conv3d_ex(const b200unet_conv_desc* desc, const b200unet_diag_ext* ext, void* stream);
/* dw fp32 [T][cip][cop].  part == NULL: dw += the gradient (atomics).  Otherwise the deterministic mode of the plans: the
 * split-K CTAs store partial sums into slots of part (part_bytes long), *splits is set to the number of slots, and a second
 * kernel writes dw = their sum in a fixed order. */
int b200unet_diag_wgrad_ex(const b200unet_tensor* a, const b200unet_tensor* dy, int ksz, int stride, int cip, int cop,
                           const b200unet_diag_ext* ext, float* part, size_t part_bytes, int* splits, float* dw, void* stream);
/* dbias[c] = sum of dy over the visible voxels (overwritten), in a fixed order: per-block partial sums into scratch
 * (b200unet_diag_bias_grad_scratch_bytes(dy->c) long), then their sum */
int b200unet_diag_bias_grad(const b200unet_tensor* dy, const b200unet_diag_ext* ext, float* scratch, float* dbias, void* stream);
size_t b200unet_diag_bias_grad_scratch_bytes(int c);
/* b200unet_gn_bwd with the per-(n, c) dropout scale [n][x->c] the plans apply to dx (NULL = none) */
int b200unet_diag_gn_bwd(const b200unet_tensor* dz, const b200unet_tensor* x, const float* coef, const double* bstats, const float* gamma,
                         int c, int groups, float* dgamma, float* dbeta, const b200unet_tensor* add1, const b200unet_tensor* add2,
                         const b200unet_tensor* dx, const float* scale, void* stream);
/* the 1x1x1 head forward of b200unet_head_fwd with a per-output bias (NULL = none), as the plans run it */
int b200unet_diag_head_fwd(const b200unet_tensor* x, const float* w, const float* bias, int n_out, int act, float* logits, void* stream);
/* b200unet_head_bwd with the fused bias gradient the plans take at 9..128 outputs: dbias[o] = sum of dlogits over n and the voxels
 * (overwritten; NULL = none, which 1..8 outputs require).  scratch: b200unet_head_bwd_scratch_bytes(n_out, x->c), owned by the
 * caller, so that a test can see which weight- and bias-gradient slots the tensor-core backward writes */
int b200unet_diag_head_bwd(const b200unet_tensor* x, const float* w, int n_out, const float* dlogits, const b200unet_tensor* dx, float* dw,
                           float* dbias, float* scratch, void* stream);
/* dbias[o] = sum of dlogits [n][n_out][spatial] over n and the voxels (overwritten), 1..32 outputs; scratch: 128 * n_out doubles */
int b200unet_diag_head_dbias(const float* dlogits, int n, int n_out, int64_t spatial, float* scratch, float* dbias, void* stream);
/* the network input NCDHW fp32 [n][c][out.d * out.h * out.w] -> NDHWC bf16 out (out->c = 8 or 16, the channels from c on stored
 * as 0); stats != NULL: also += the fp64 (sum, sumsq) of each of the c channels, [n][stats_ld][2] */
int b200unet_diag_input_pack(const float* x, int c, const b200unet_tensor* out, double* stats, int stats_ld, void* stream);
/* the gradient of the network input, NCDHW fp32 [n][c][r.d * r.h * r.w]: dx = (A dz + E x + F) + r over its c <= 16 channels,
 * A from coef [n][coef_ld][4], (E, F) from coef2 [n][coef_ld][2]; dz == NULL: dx = r (x, coef and coef2 are then unused) */
int b200unet_diag_input_grad(const b200unet_tensor* dz, const b200unet_tensor* x, const float* coef, const float* coef2, int coef_ld,
                             const b200unet_tensor* r, int c, float* dx, void* stream);

/* the raw distance fields behind b200unet_hausdorff_dt_weight: pred_field / target_field DEVICE fp32 [n][c'][d*h*w] =
 * edt(mask) + edt(~mask) of the prediction and target masks (0 for an empty or full mask); either NULL = not computed.  scratch:
 * b200unet_hausdorff_dt_scratch_bytes() bytes */
int b200unet_diag_hausdorff_dt_fields(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c, int d,
                                      int h, int w, void* scratch, float* pred_field, float* target_field, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200UNET_DIAG_H_ */
