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
} b200unet_diag_ext;

/* kernel kinds of b200unet_conv_route */
#define B200UNET_CONV_TAP 0      /* per-tap streaming tiles */
#define B200UNET_CONV_HALO 1     /* one halo box per K chunk for an 8 x 16 x 1 output tile */
#define B200UNET_CONV_CLASS1 2   /* parity classes: data gradient of a 3x3x3 stride-2 convolution */
#define B200UNET_CONV_CLASS2 3   /* parity classes: ConvTranspose3d with kernel = stride = 2 */

typedef struct b200unet_conv_route {
  int32_t kind;
  int32_t bn, kc;                 /* output channels per CTA, input channels per K chunk */
  int32_t kchunks[2];             /* K chunks of each source */
  int32_t npass;                  /* 1 bf16, 3 split precision */
  int32_t cls_pair;               /* class mode in bf16: the two W-parity classes share one store */
  int32_t tw, th, td;             /* output voxel tile (class mode: of one parity class) */
  int32_t grid[3];
  int32_t stages, blocks_per_sm, smem_bytes;   /* of the kernel's compile-time configuration */
} b200unet_conv_route;

/* kernel kinds of b200unet_wgrad_route */
#define B200UNET_WGRAD_SIMT 0    /* 1x1x1 with 8 or 16 input channels, register tiles, atomics only */
#define B200UNET_WGRAD_TAP 1     /* tensor cores, one TMA box per (tap, channel chunk) */
#define B200UNET_WGRAD_HALO 2    /* tensor cores, one halo box per 8 x 16 x 1 voxel tile */

typedef struct b200unet_wgrad_route {
  int32_t kind;
  int32_t ci8;                    /* SIMT: input channels / 8 */
  int32_t cb, bn, qt;             /* input channels per M box, output channels per N tile, M tiles per CTA */
  int32_t groups, cotiles, kblocks, splits, npass;
  int32_t tw, th, td;
  int64_t part_bytes;             /* deterministic mode: splits * taps * cip * cop * 4, the partial-sum buffer it fills */
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
 * split-K CTAs store partial sums into part (part_bytes long), *splits is set to their number, and a second kernel writes
 * dw = their sum in a fixed order. */
int b200unet_diag_wgrad_ex(const b200unet_tensor* a, const b200unet_tensor* dy, int ksz, int stride, int cip, int cop,
                           const b200unet_diag_ext* ext, float* part, size_t part_bytes, int* splits, float* dw, void* stream);
/* dbias[c] = sum of dy over the visible voxels (overwritten) */
int b200unet_diag_bias_grad(const b200unet_tensor* dy, const b200unet_diag_ext* ext, float* dbias, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200UNET_DIAG_H_ */
