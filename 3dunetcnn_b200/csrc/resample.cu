// Resample a prediction onto the grid of the image file it came from (MONAI ResampleToMatch as the reference calls it after
// inference: unet3d/predict/volumetric.py:135-137,168-170, paths relative to /root/reference).  HBM-bound, NCDHW fp32.
//
//   k_resample_to_grid   one thread per target voxel (d, h, w): the source index M (d, h, w, 1) in fp64 from the 3x4 index
//                        affine, then every channel: trilinear (the 8 corners' offsets and fp32 weights computed once) or nearest
//                        (round half to even), each channel plane written coalesced.
//
// Border padding only: the source coordinate is clamped to [0, size-1] on every axis (ResampleToMatch's default).
#include "kernels.h"
#include "resample.cuh"

namespace b200 {

static constexpr int kResThreads = 256;

struct ResGrid {
  int sd, sh, sw;        // source extents
  int dd, dh, dw;        // target extents
  long long ss, ds;      // voxels per channel plane of the source / target, each < 2^31
};

template <int NEAREST>
__global__ void __launch_bounds__(kResThreads) k_resample_to_grid(const float* __restrict__ src, int C, ResGrid g,
                                                                   IndexAffine m, float* __restrict__ dst) {
  const long long v = (long long)blockIdx.x * kResThreads + threadIdx.x;
  if (v >= g.ds) return;
  const unsigned u = (unsigned)v, hw = (unsigned)g.dh * (unsigned)g.dw;   // S < 2^31: 32-bit index arithmetic
  const int d = (int)(u / hw);
  const int h = (int)((u - d * hw) / (unsigned)g.dw);
  const int w = (int)(u - d * hw - h * (unsigned)g.dw);
  const double fd = (double)d, fh = (double)h, fw = (double)w;
  const double* a = m.m;
  const double xd = fma(a[0], fd, fma(a[1], fh, fma(a[2], fw, a[3])));
  const double xh = fma(a[4], fd, fma(a[5], fh, fma(a[6], fw, a[7])));
  const double xw = fma(a[8], fd, fma(a[9], fh, fma(a[10], fw, a[11])));
  if (NEAREST) {
    // clamp, then round half to even, as grid_sample's nearest mode with border padding
    const int id = (int)rint(fmin(fmax(xd, 0.0), (double)(g.sd - 1)));
    const int ih = (int)rint(fmin(fmax(xh, 0.0), (double)(g.sh - 1)));
    const int iw = (int)rint(fmin(fmax(xw, 0.0), (double)(g.sw - 1)));
    const int o = (id * g.sh + ih) * g.sw + iw;
#pragma unroll 4
    for (int c = 0; c < C; ++c) dst[(long long)c * g.ds + v] = __ldg(src + (long long)c * g.ss + o);
  } else {
    const Trilinear t = trilinear_corners(xd, xh, xw, g.sd, g.sh, g.sw, 1);
#pragma unroll 4
    for (int c = 0; c < C; ++c) dst[(long long)c * g.ds + v] = trilinear_sample(src + (long long)c * g.ss, t);
  }
}

int launch_resample_to_grid(const float* src, int C, int sd, int sh, int sw, const IndexAffine& m, int mode, float* dst, int dd,
                            int dh, int dw, cudaStream_t st) {
  B200_REQUIRE(src && dst, E_INVALID, "resample_to_grid: null argument");
  B200_REQUIRE(C >= 1 && C <= B200_MAX_LABEL_CHANNELS, E_UNSUPPORTED, "resample_to_grid: 1..%d channels, got %d",
               B200_MAX_LABEL_CHANNELS, C);
  B200_REQUIRE(mode == 0 || mode == 1, E_UNSUPPORTED, "resample_to_grid: mode 0 (trilinear) or 1 (nearest), got %d", mode);
  const long long ss = (long long)sd * sh * sw, ds = (long long)dd * dh * dw;
  B200_REQUIRE(sd >= 1 && sh >= 1 && sw >= 1 && dd >= 1 && dh >= 1 && dw >= 1 && ss < (1LL << 31) && ds < (1LL << 31), E_UNSUPPORTED,
               "resample_to_grid: extents >= 1 and fewer than 2^31 voxels per channel (source %dx%dx%d, target %dx%dx%d)", sd, sh, sw,
               dd, dh, dw);
  for (int k = 0; k < 12; ++k)
    B200_REQUIRE(isfinite(m.m[k]), E_INVALID, "resample_to_grid: index affine entry %d is not finite", k);
  const ResGrid g{sd, sh, sw, dd, dh, dw, ss, ds};
  const unsigned blocks = (unsigned)((ds + kResThreads - 1) / kResThreads);
  if (mode == 1)
    k_resample_to_grid<1><<<blocks, kResThreads, 0, st>>>(src, C, g, m, dst);
  else
    k_resample_to_grid<0><<<blocks, kResThreads, 0, st>>>(src, C, g, m, dst);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

}  // namespace b200
