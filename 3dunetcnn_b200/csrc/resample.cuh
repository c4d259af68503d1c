// Trilinear corner and weight logic shared by the resampling kernels (augment.cu, resample.cu).  Index coordinates: voxel
// centres sit on integers, as grid_sample(align_corners=False) on index coordinates.  The source coordinate may be fp32
// (augment) or fp64 (resample to a file's grid); the weights are fp32 either way.
#pragma once
#include <cuda_runtime.h>

namespace b200 {

// source coordinate on one axis -> the two corner indices and the weight of the upper one, corners outside the volume
// flagged by ok0 / ok1 (zeros padding); border clamps the coordinate to [0, n-1] first
template <typename T>
__device__ __forceinline__ void trilinear_axis(T x, int n, int border, int& i0, int& i1, float& f, bool& ok0, bool& ok1) {
  if constexpr (sizeof(T) == sizeof(float)) {
    if (border) x = fminf(fmaxf(x, 0.f), (float)(n - 1));
    const float fl = floorf(x);
    f = x - fl;
    i0 = (int)fl;
  } else {
    if (border) x = fmin(fmax(x, 0.0), (double)(n - 1));
    const double fl = floor(x);
    f = (float)(x - fl);
    i0 = (int)fl;
  }
  i1 = i0 + 1;
  ok0 = i0 >= 0 && i0 < n;
  ok1 = i1 >= 0 && i1 < n;
}

// the 8 corners of one sample point in a (D, H, W) plane of fewer than 2^31 voxels
struct Trilinear {
  float wt[8];
  int off[8];
  bool ok[8];
  bool any;   // some corner is read (false only with zeros padding, every corner outside)
};

template <typename T>
__device__ __forceinline__ Trilinear trilinear_corners(T sd, T sh, T sw, int D, int H, int W, int border) {
  Trilinear t;
  int d0, d1, h0, h1, w0, w1;
  float ad, ah, aw;
  bool od0, od1, oh0, oh1, ow0, ow1;
  trilinear_axis(sd, D, border, d0, d1, ad, od0, od1);
  trilinear_axis(sh, H, border, h0, h1, ah, oh0, oh1);
  trilinear_axis(sw, W, border, w0, w1, aw, ow0, ow1);
  // border: the upper corner of the last plane carries weight 0; read the last plane instead of past it
  if (border) { d1 = min(d1, D - 1); h1 = min(h1, H - 1); w1 = min(w1, W - 1); od1 = oh1 = ow1 = true; }
  const float bd = 1.f - ad, bh = 1.f - ah, bw = 1.f - aw;
  t.wt[0] = bd * bh * bw; t.wt[1] = bd * bh * aw; t.wt[2] = bd * ah * bw; t.wt[3] = bd * ah * aw;
  t.wt[4] = ad * bh * bw; t.wt[5] = ad * bh * aw; t.wt[6] = ad * ah * bw; t.wt[7] = ad * ah * aw;
  // a corner counts when it lies inside the volume and has a non-zero weight: corners of weight 0 are not read, so a
  // flip copies every value bit for bit (-0.0, inf and NaN included) and an inf beside a voxel does not leak into it
  t.ok[0] = od0 && oh0 && ow0; t.ok[1] = od0 && oh0 && ow1; t.ok[2] = od0 && oh1 && ow0; t.ok[3] = od0 && oh1 && ow1;
  t.ok[4] = od1 && oh0 && ow0; t.ok[5] = od1 && oh0 && ow1; t.ok[6] = od1 && oh1 && ow0; t.ok[7] = od1 && oh1 && ow1;
  t.any = false;
#pragma unroll
  for (int k = 0; k < 8; ++k) { t.ok[k] = t.ok[k] && t.wt[k] != 0.f; t.any = t.any || t.ok[k]; }
  const int dd[2] = {d0, d1}, hh[2] = {h0, h1}, ww[2] = {w0, w1};
#pragma unroll
  for (int k = 0; k < 8; ++k) t.off[k] = t.ok[k] ? (dd[k >> 2] * H + hh[(k >> 1) & 1]) * W + ww[k & 1] : 0;
  return t;
}

// the weighted sum of the corners read from one channel plane p, in one fixed fma order
__device__ __forceinline__ float trilinear_sample(const float* __restrict__ p, const Trilinear& t) {
  float y = -0.f;                 // -0 + x == x for every x, so a single corner passes through unchanged
#pragma unroll
  for (int k = 0; k < 8; ++k)
    if (t.ok[k]) y = fmaf(t.wt[k], __ldg(p + t.off[k]), y);
  return y;
}

}  // namespace b200
