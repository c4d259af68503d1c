/* libb200unet diagnostics -- NOT part of the product ABI (include/b200unet.h).
 *
 * A SIMT cross-check convolution used by tools/gpu_diag.py while the kernels were developed.  It lives in the same shared
 * object so that it sees the same build flags, but nothing in the model / training / inference path calls it.
 */
#ifndef B200UNET_DIAG_H_
#define B200UNET_DIAG_H_
#include "b200unet.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- SIMT direct convolution on the same packed operands (cross-check only; not used by the model path) */
int b200unet_conv3d_simt(const b200unet_tensor* x, const void* w_hi, const void* w_lo, int ksz, int stride,
                         const b200unet_tensor* y, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200UNET_DIAG_H_ */
