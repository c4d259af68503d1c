// Random spatial + intensity augmentation of a training batch on the device (HBM-bound, NCDHW).  Paths relative to
// /root/reference: unet3d/datasets/segmentation.py:72-94 (MONAI RandFlipd / RandRotated with lazy=True, NormalizeIntensityd,
// RandScaleIntensityd / RandShiftIntensityd).
//
//   k_aug_resample   pass 1: one thread per output voxel maps (d, h, w) through the sample's 3x4 index-space affine to a source
//                    position and samples every image channel there (trilinear) and every label channel (nearest); the same
//                    pass writes per-block fp64 (sum, sumsq, count) partials of the resampled image per (n, c).  The source is
//                    the batch itself on the output grid, or per sample a pointer and extents of its own (foreground.cu)
//   k_aug_stats      fixed-order reduction of the partials -> stats [n][c][3]
//   k_aug_apply      pass 2, in place: y = ((x - mean) / std) * a + b per (n, c)
//
// Padding follows torch.nn.functional.grid_sample(align_corners=False) on index coordinates: border clamps the source
// coordinate to [0, size-1], zeros gives out-of-range corners weight 0 (labels 0); nearest rounds half to even.
#include "kernels.h"
#include "resample.cuh"

namespace b200 {

static constexpr int kAugThreads = 256;
static constexpr int kAugMaxBlocks = 1024;    // partial slots per sample
static constexpr int kAugVoxelsPerBlock = 2048;

// blocks per sample of k_aug_resample: a function of the shape alone, so the scratch size is known before the launch
static int aug_blocks(long long S) {
  long long b = (S + kAugVoxelsPerBlock - 1) / kAugVoxelsPerBlock;
  return (int)(b < 1 ? 1 : b > kAugMaxBlocks ? kAugMaxBlocks : b);
}

size_t augment_scratch_bytes(int N, int C, long long S) {
  if (N < 1 || C < 1 || C > B200_AUG_MAX_CHANNELS || S < 1 || S >= (1LL << 31)) {
    set_error("augment: 1..%d image channels, n >= 1 and 1 <= d*h*w < 2^31 (n=%d c=%d spatial=%lld)", B200_AUG_MAX_CHANNELS, N, C, S);
    return 0;
  }
  return sizeof(double) * 3 * (size_t)N * C * (1 + (size_t)aug_blocks(S));
}

struct AugDims {
  int D, H, W;
  long long S;
};

// g: the output grid.  samples == nullptr: sample n reads img / lab at n * C * g.S / n * L * g.S on the same grid; otherwise
// samples[n] gives its own source pointers and extents (a batch of different sizes resampled onto one grid)
template <int CM>
__global__ void __launch_bounds__(kAugThreads) k_aug_resample(const float* __restrict__ img, const uint8_t* __restrict__ lab,
                                                               const AugSample* __restrict__ samples, int C, int L, AugDims g,
                                                               const float* __restrict__ affine, int border, int nonzero,
                                                               float* __restrict__ out, uint8_t* __restrict__ lout,
                                                               double* __restrict__ part) {
  const int n = blockIdx.y;
  const int nb = gridDim.x;
  const long long per = (g.S + nb - 1) / nb;
  const long long v0 = (long long)blockIdx.x * per;
  const long long v1 = v0 + per < g.S ? v0 + per : g.S;
  float m[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) m[k] = __ldg(affine + n * 12 + k);
  const float* src;
  const uint8_t* lp;
  int SD, SH, SW;
  if (samples) {
    const AugSample sm = samples[n];
    src = sm.img; lp = sm.lab;
    SD = (int)sm.d; SH = (int)sm.h; SW = (int)sm.w;
  } else {
    src = img + (long long)n * C * g.S;
    lp = L > 0 ? lab + (long long)n * L * g.S : nullptr;
    SD = g.D; SH = g.H; SW = g.W;
  }
  const long long SS = (long long)SD * SH * SW;     // source channel stride
  float* dst = out + (long long)n * C * g.S;

  double s[CM], q[CM];
  unsigned cnt[CM];
#pragma unroll
  for (int c = 0; c < CM; ++c) { s[c] = 0.0; q[c] = 0.0; cnt[c] = 0u; }

  for (long long v = v0 + threadIdx.x; v < v1; v += kAugThreads) {
    const unsigned u = (unsigned)v, hw = (unsigned)g.H * (unsigned)g.W;   // S < 2^31: 32-bit index arithmetic
    const int d = (int)(u / hw);
    const int h = (int)((u - d * hw) / (unsigned)g.W);
    const int w = (int)(u - d * hw - h * (unsigned)g.W);
    const float fd = (float)d, fh = (float)h, fw = (float)w;
    // source index = M (d, h, w) + t, one fixed fma order
    const float sd = fmaf(m[0], fd, fmaf(m[1], fh, fmaf(m[2], fw, m[3])));
    const float sh = fmaf(m[4], fd, fmaf(m[5], fh, fmaf(m[6], fw, m[7])));
    const float sw = fmaf(m[8], fd, fmaf(m[9], fh, fmaf(m[10], fw, m[11])));

    const Trilinear t = trilinear_corners(sd, sh, sw, SD, SH, SW, border);   // offsets within one plane: S < 2^31
#pragma unroll
    for (int c = 0; c < CM; ++c) {
      if (c < C) {
        float y = trilinear_sample(src + (long long)c * SS, t);
        if (!t.any) y = 0.f;            // every corner outside the volume (zeros padding)
        dst[(long long)c * g.S + v] = y;
        if (!nonzero || y != 0.f) { s[c] += y; q[c] += (double)y * y; cnt[c] += 1u; }
      }
    }
    if (L > 0) {
      // nearest: round half to even of the (clamped) coordinate, as grid_sample's nearest mode
      const float rd = rintf(border ? fminf(fmaxf(sd, 0.f), (float)(SD - 1)) : sd);
      const float rh = rintf(border ? fminf(fmaxf(sh, 0.f), (float)(SH - 1)) : sh);
      const float rw = rintf(border ? fminf(fmaxf(sw, 0.f), (float)(SW - 1)) : sw);
      const bool in = rd >= 0.f && rd < (float)SD && rh >= 0.f && rh < (float)SH && rw >= 0.f && rw < (float)SW;
      const int o = in ? ((int)rd * SH + (int)rh) * SW + (int)rw : 0;
      uint8_t* lo = lout + (long long)n * L * g.S;
      for (int c = 0; c < L; ++c) lo[(long long)c * g.S + v] = in ? __ldg(lp + (long long)c * SS + o) : (uint8_t)0;
    }
  }

  // block partials in a fixed order: warp butterfly, then warp 0 adds the warps' sums in index order
  __shared__ double red[3][kAugThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < CM; ++c) {
    if (c >= C) break;                // C is uniform over the block: every thread leaves at the same c
    double a = s[c], b = q[c], k = (double)cnt[c];
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o);
      b += __shfl_xor_sync(0xffffffffu, b, o);
      k += __shfl_xor_sync(0xffffffffu, k, o);
    }
    if (lane == 0) { red[0][wid] = a; red[1][wid] = b; red[2][wid] = k; }
    __syncthreads();
    if (threadIdx.x == 0) {
      double ta = 0, tb = 0, tk = 0;
      for (int i = 0; i < kAugThreads / 32; ++i) { ta += red[0][i]; tb += red[1][i]; tk += red[2][i]; }
      double* pp = part + (((long long)n * nb + blockIdx.x) * C + c) * 3;
      pp[0] = ta; pp[1] = tb; pp[2] = tk;
    }
    __syncthreads();
  }
}

// stats[n][c] = sum over the blocks of part[n][blk][c], one block per (n, c): strided per-thread sums, then a fixed tree
__global__ void __launch_bounds__(kAugThreads) k_aug_stats(const double* __restrict__ part, int C, int nb, double* __restrict__ stats) {
  const int n = blockIdx.x / C, c = blockIdx.x % C;
  double a = 0, b = 0, k = 0;
  for (int i = threadIdx.x; i < nb; i += kAugThreads) {
    const double* pp = part + (((long long)n * nb + i) * C + c) * 3;
    a += pp[0]; b += pp[1]; k += pp[2];
  }
  __shared__ double sh[3][kAugThreads];
  sh[0][threadIdx.x] = a; sh[1][threadIdx.x] = b; sh[2][threadIdx.x] = k;
  __syncthreads();
  for (int o = kAugThreads / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o)
      for (int j = 0; j < 3; ++j) sh[j][threadIdx.x] += sh[j][threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0)
    for (int j = 0; j < 3; ++j) stats[(long long)blockIdx.x * 3 + j] = sh[j][0];
}

// y = ((x - mean) / std) * a + b on plane (n, c) = blockIdx.y; normalize == 0: y = x * a + b.  With nonzero, zero voxels skip the
// z-score (MONAI NormalizeIntensity) but not the scale / shift.  Statistics of the group: channel c, or all C channels of n.
__global__ void __launch_bounds__(kAugThreads) k_aug_apply(float* __restrict__ x, int C, long long S, int vec4, int normalize, int nonzero,
                                                            int channel_wise, const double* __restrict__ stats,
                                                            const float* __restrict__ coef) {
  const int n = blockIdx.y / C, c = blockIdx.y % C;
  float m = 0.f, inv = 1.f;
  if (normalize) {
    double ts = 0, tq = 0, tk = 0;
    for (int j = channel_wise ? c : 0; j < (channel_wise ? c + 1 : C); ++j) {
      const double* st = stats + ((long long)n * C + j) * 3;
      ts += st[0]; tq += st[1]; tk += st[2];
    }
    const double mean = tk > 0 ? ts / tk : 0.0;
    double var = tk > 0 ? tq / tk - mean * mean : 0.0;
    if (var < 0) var = 0;
    double sd = sqrt(var);
    if (sd == 0.0) sd = 1.0;
    m = (float)mean;
    inv = (float)(1.0 / sd);
  }
  const float a = __ldg(coef + (long long)blockIdx.y * 2), b = __ldg(coef + (long long)blockIdx.y * 2 + 1);
  if (!normalize && a == 1.f && b == 0.f) return;   // nothing drawn for this plane: leave it as it is (fmaf would turn -0 into +0)
  float* p = x + (long long)blockIdx.y * S;
  auto f = [&](float v) -> float {
    const float z = (normalize && (!nonzero || v != 0.f)) ? (v - m) * inv : v;
    return fmaf(z, a, b);
  };
  if (vec4) {
    float4* p4 = reinterpret_cast<float4*>(p);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < S / 4; i += (long long)gridDim.x * blockDim.x) {
      float4 v = p4[i];
      v.x = f(v.x); v.y = f(v.y); v.z = f(v.z); v.w = f(v.w);
      p4[i] = v;
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < S; i += (long long)gridDim.x * blockDim.x) p[i] = f(p[i]);
  }
}

static int augment_resample(const float* img, const uint8_t* lab, const AugSample* samples, int N, int C, int L, int D, int H, int W,
                            const float* affine, int padding, int nonzero, float* img_out, uint8_t* lab_out, void* scratch,
                            cudaStream_t st) {
  B200_REQUIRE(affine && img_out && scratch, E_INVALID, "augment_resample: null argument");
  B200_REQUIRE(L == 0 || lab_out, E_INVALID, "augment_resample: %d label channels but no label output", L);
  B200_REQUIRE(N >= 1 && N <= 65535 && D >= 1 && H >= 1 && W >= 1 && L >= 0, E_INVALID,
               "augment_resample: bad shape n=%d l=%d %dx%dx%d", N, L, D, H, W);
  B200_REQUIRE(padding == 0 || padding == 1, E_UNSUPPORTED, "augment_resample: padding 0 (border) or 1 (zeros), got %d", padding);
  const long long S = (long long)D * H * W;
  if (augment_scratch_bytes(N, C, S) == 0) return E_UNSUPPORTED;
  AugDims g{D, H, W, S};
  const dim3 grid(aug_blocks(S), N);
  double* part = reinterpret_cast<double*>(scratch) + (size_t)N * C * 3;
  const int border = padding == 0;
  if (C <= 4)
    k_aug_resample<4><<<grid, kAugThreads, 0, st>>>(img, lab, samples, C, L, g, affine, border, nonzero, img_out, lab_out, part);
  else
    k_aug_resample<B200_AUG_MAX_CHANNELS><<<grid, kAugThreads, 0, st>>>(img, lab, samples, C, L, g, affine, border, nonzero, img_out,
                                                                       lab_out, part);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

int launch_augment_resample(const float* img, const uint8_t* lab, int N, int C, int L, int D, int H, int W, const float* affine,
                            int padding, int nonzero, float* img_out, uint8_t* lab_out, void* scratch, cudaStream_t st) {
  B200_REQUIRE(img, E_INVALID, "augment_resample: null argument");
  B200_REQUIRE(L == 0 || lab, E_INVALID, "augment_resample: %d label channels but no label tensors", L);
  return augment_resample(img, lab, nullptr, N, C, L, D, H, W, affine, padding, nonzero, img_out, lab_out, scratch, st);
}

int launch_augment_resample_samples(const AugSample* samples, int N, int C, int L, int D, int H, int W, const float* affine,
                                    int padding, int nonzero, float* img_out, uint8_t* lab_out, void* scratch, cudaStream_t st) {
  B200_REQUIRE(samples, E_INVALID, "augment_resample_samples: null sample table");
  return augment_resample(nullptr, nullptr, samples, N, C, L, D, H, W, affine, padding, nonzero, img_out, lab_out, scratch, st);
}

int launch_augment_intensity(float* img, int N, int C, long long S, int normalize, int nonzero, int channel_wise, const float* coef,
                             void* scratch, cudaStream_t st) {
  B200_REQUIRE(img && coef && scratch, E_INVALID, "augment_intensity: null argument");
  if (augment_scratch_bytes(N, C, S) == 0) return E_UNSUPPORTED;
  B200_REQUIRE(N <= 65535 / C, E_INVALID, "augment_intensity: n * c = %d planes, at most 65535", N * C);
  double* stats = reinterpret_cast<double*>(scratch);
  if (normalize) {
    k_aug_stats<<<N * C, kAugThreads, 0, st>>>(stats + (size_t)N * C * 3, C, aug_blocks(S), stats);
    B200_CHECK_CUDA(cudaGetLastError());
  }
  long long chunks = ((S + 3) / 4 + kAugThreads * 4 - 1) / (kAugThreads * 4);
  const long long cap = (132LL * 8 + N * C - 1) / (N * C);
  if (chunks > cap) chunks = cap;
  if (chunks < 1) chunks = 1;
  // float4 when every plane starts on a 16-byte boundary
  const int vec4 = (S & 3) == 0 && (reinterpret_cast<uintptr_t>(img) & 15) == 0;
  k_aug_apply<<<dim3((unsigned)chunks, N * C), kAugThreads, 0, st>>>(img, C, S, vec4, normalize, nonzero, channel_wise, stats, coef);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

}  // namespace b200
