// Foreground box of each training sample and the one source map of crop + resize + augmentation (HBM-bound).  Paths relative
// to /root/reference: unet3d/datasets/segmentation.py:55-70 (MONAI CropForegroundD with utils/threshold.py's
// percentile_threshold, then ResizeD, composed lazily with the spatial augmentations).
//
//   k_fg_hist / k_fg_scan   exact radix select per (sample, channel): three histogram passes over order-preserving uint32 keys
//                           (11, 11, 10 bits), each followed by a one-block-per-plane scan that picks the bin holding each of
//                           the two ranks numpy's linear percentile interpolates between; the last scan interpolates thr
//   k_fg_box                mask any_c(x_c > thr_c) and its per-axis first / last index, integer atomicMax (exact, any order)
//   k_fg_compose            box (margin, clipping, empty -> whole volume) composed with the resize scale and the drawn affine
//
// Every kernel reads the samples through a DEVICE table of pointers and extents, so one launch covers a batch of different
// sizes and nothing is read back to the host.
#include "kernels.h"

namespace b200 {

static constexpr int kFgThreads = 256;
static constexpr int kFgBins = 2048;                  // 11-bit digits; the last pass uses 10 bits
static constexpr int kFgUnroll = 4;                   // loads in flight per thread
static constexpr int kFgTargetBlocks = 132 * 8;       // blocks per histogram / box launch, over all planes

// digit of pass 0, 1, 2: key bits 31..21, 20..10, 9..0
__host__ __device__ constexpr int fg_shift(int pass) { return pass == 0 ? 21 : pass == 1 ? 10 : 0; }
__host__ __device__ constexpr int fg_bits(int pass) { return pass == 2 ? 10 : 11; }

struct FgPlane {
  unsigned prefix[2];   // key bits fixed so far for the lower and the upper rank
  unsigned rank[2];     // ranks left within that prefix
  int nan;              // the plane holds a NaN: thr = NaN
  int pad;
};

static size_t fg_hist_bytes(int P) { return sizeof(unsigned) * 2 * kFgBins * (size_t)P; }

size_t foreground_scratch_bytes(int N, int C) {
  if (N < 1 || N > 65535 || C < 1 || C > B200_AUG_MAX_CHANNELS) {
    set_error("foreground: 1..%d channels and 1..65535 samples (n=%d c=%d)", B200_AUG_MAX_CHANNELS, N, C);
    return 0;
  }
  if (N * C > 65535) {   // k_fg_hist puts the planes on gridDim.y
    set_error("foreground: n * c = %d planes, at most 65535 (n=%d c=%d)", N * C, N, C);
    return 0;
  }
  const int P = N * C;
  return fg_hist_bytes(P) + sizeof(FgPlane) * (size_t)P + sizeof(int) * 6 * (size_t)N;
}

// float -> uint32 whose unsigned order is the float order; -0 takes the key of +0 (numpy's sort does not order them)
__device__ __forceinline__ unsigned fg_key(float x) {
  unsigned u = __float_as_uint(x);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float fg_value(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k ^ 0x80000000u) : ~k); }

// one pass: per plane (blockIdx.y), histogram of the digit of the keys that carry each rank's prefix; while the two ranks
// share their prefix one histogram serves both.  NaNs are counted out and flag the plane.
__global__ void __launch_bounds__(kFgThreads) k_fg_hist(const AugSample* __restrict__ samples, int C, int pass,
                                                        FgPlane* __restrict__ planes, unsigned* __restrict__ hist) {
  __shared__ unsigned sh[2 * kFgBins];
  const int plane = blockIdx.y;
  const AugSample sm = samples[plane / C];
  const long long S = sm.d * sm.h * sm.w;
  const long long per = (S + gridDim.x - 1) / gridDim.x;
  const long long v0 = (long long)blockIdx.x * per;
  const long long v1 = v0 + per < S ? v0 + per : S;
  if (v0 >= S) return;                                 // uniform over the block: a small plane uses fewer blocks
  for (int i = threadIdx.x; i < 2 * kFgBins; i += kFgThreads) sh[i] = 0u;
  const int shift = fg_shift(pass);
  const unsigned dmask = (1u << fg_bits(pass)) - 1u;
  const unsigned mask = pass == 0 ? 0u : ~((1u << (shift + fg_bits(pass))) - 1u);
  const unsigned p0 = pass == 0 ? 0u : planes[plane].prefix[0];
  const unsigned p1 = pass == 0 ? 0u : planes[plane].prefix[1];
  const bool two = p0 != p1;
  const float* x = sm.img + (long long)(plane % C) * S;
  __syncthreads();
  bool nan = false;
  for (long long base = v0; base < v1; base += kFgThreads * kFgUnroll) {   // every lane runs the same iterations
    float f[kFgUnroll];
#pragma unroll
    for (int j = 0; j < kFgUnroll; ++j) {
      const long long v = base + j * kFgThreads + threadIdx.x;
      f[j] = v < v1 ? __ldg(x + v) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < kFgUnroll; ++j) {
      const long long v = base + j * kFgThreads + threadIdx.x;
      unsigned bin = 0xffffffffu;
      if (v < v1) {
        if (f[j] != f[j]) {
          nan = true;
        } else {
          const unsigned k = fg_key(f[j]);
          if ((k & mask) == p0) bin = (k >> shift) & dmask;
          else if (two && (k & mask) == p1) bin = kFgBins + ((k >> shift) & dmask);
        }
      }
      // heavy ties (MRI volumes are mostly exact zeros): one shared atomic per distinct bin of the warp
      const unsigned peers = __match_any_sync(0xffffffffu, bin);
      if (bin != 0xffffffffu && (int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&sh[bin], (unsigned)__popc(peers));
    }
  }
  if (nan) planes[plane].nan = 1;
  __syncthreads();
  unsigned* gh = hist + (size_t)plane * 2 * kFgBins;
  for (int i = threadIdx.x; i < (two ? 2 : 1) * kFgBins; i += kFgThreads)
    if (sh[i]) atomicAdd(gh + i, sh[i]);
}

// one block per plane: find the bin of each rank in the pass's histogram, fix its digit, keep the rank within the bin, zero
// the histogram for the next pass.  After the last pass both keys are complete: thr = numpy's _lerp of the two values in fp32.
__global__ void __launch_bounds__(kFgThreads) k_fg_scan(int pass, const long long* __restrict__ ranks, const float* __restrict__ gamma,
                                                        FgPlane* __restrict__ planes, unsigned* __restrict__ hist,
                                                        float* __restrict__ thr) {
  constexpr int kPer = kFgBins / kFgThreads;
  __shared__ unsigned wsum[kFgThreads / 32];
  __shared__ unsigned res[2][2];
  const int plane = blockIdx.x;
  unsigned pre[2], rk[2];
  if (pass == 0) {
    pre[0] = pre[1] = 0u;
    rk[0] = (unsigned)ranks[plane * 2];
    rk[1] = (unsigned)ranks[plane * 2 + 1];
  } else {
    pre[0] = planes[plane].prefix[0]; pre[1] = planes[plane].prefix[1];
    rk[0] = planes[plane].rank[0]; rk[1] = planes[plane].rank[1];
  }
  const bool two = pre[0] != pre[1];
  unsigned* gh = hist + (size_t)plane * 2 * kFgBins;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x < 2) { res[threadIdx.x][0] = pre[threadIdx.x]; res[threadIdx.x][1] = rk[threadIdx.x]; }   // kept if not found
  __syncthreads();
  for (int t = 0; t < 2; ++t) {
    const unsigned* h = gh + (two ? t : 0) * kFgBins + threadIdx.x * kPer;
    unsigned own[kPer], sum = 0;
#pragma unroll
    for (int j = 0; j < kPer; ++j) { own[j] = h[j]; sum += own[j]; }
    // exclusive prefix of the per-thread sums over the block
    unsigned inc = sum;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += y;
    }
    if (lane == 31) wsum[wid] = inc;
    __syncthreads();
    unsigned before = inc - sum;
    for (int i = 0; i < wid; ++i) before += wsum[i];
    if (sum > 0 && before <= rk[t] && rk[t] - before < sum) {
      unsigned r = rk[t] - before;
#pragma unroll
      for (int j = 0; j < kPer; ++j) {
        if (r < own[j]) {
          res[t][0] = pre[t] | ((unsigned)(threadIdx.x * kPer + j) << fg_shift(pass));
          res[t][1] = r;
          break;
        }
        r -= own[j];
      }
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < 2 * kFgBins; i += kFgThreads) gh[i] = 0u;
  if (threadIdx.x == 0) {
    FgPlane& p = planes[plane];
    p.prefix[0] = res[0][0]; p.prefix[1] = res[1][0];
    p.rank[0] = res[0][1]; p.rank[1] = res[1][1];
    if (pass == 2) {
      // numpy _lerp(a, b, t) in the data's dtype: a + (b - a) t, or b - (b - a)(1 - t) where t >= 0.5; no fma contraction
      const float a = fg_value(res[0][0]), b = fg_value(res[1][0]), g = gamma[plane];
      const float diff = __fsub_rn(b, a);
      float v = g >= 0.5f ? __fsub_rn(b, __fmul_rn(diff, __fsub_rn(1.f, g))) : __fadd_rn(a, __fmul_rn(diff, g));
      if (p.nan) v = __int_as_float(0x7fffffff);
      thr[plane] = v;
    }
  }
}

__device__ __forceinline__ int fg_wmax(int v) {
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// acc[n] = max over the selected voxels of (D - d, d + 1, H - h, h + 1, W - w, w + 1): zero-initialised, 0 = nothing selected
__global__ void __launch_bounds__(kFgThreads) k_fg_box(const AugSample* __restrict__ samples, int C, const float* __restrict__ thr,
                                                       int* __restrict__ acc) {
  __shared__ float t[B200_AUG_MAX_CHANNELS];
  __shared__ int red[6][kFgThreads / 32];
  const int n = blockIdx.y;
  const AugSample sm = samples[n];
  const long long S = sm.d * sm.h * sm.w;
  const long long per = (S + gridDim.x - 1) / gridDim.x;
  const long long v0 = (long long)blockIdx.x * per;
  const long long v1 = v0 + per < S ? v0 + per : S;
  if (v0 >= S) return;
  if ((int)threadIdx.x < C) t[threadIdx.x] = thr ? thr[n * C + threadIdx.x] : 0.f;
  __syncthreads();
  const int D = (int)sm.d, H = (int)sm.h, W = (int)sm.w;
  int m[6] = {0, 0, 0, 0, 0, 0};
  for (long long v = v0 + threadIdx.x; v < v1; v += kFgThreads) {
    bool sel = false;
    for (int c = 0; c < C && !sel; ++c) sel = __ldg(sm.img + c * S + v) > t[c];   // NaN > x and x > NaN are false
    if (sel) {
      const unsigned u = (unsigned)v, hw = (unsigned)H * (unsigned)W;                // S < 2^31
      const int d = (int)(u / hw);
      const int h = (int)((u - d * hw) / (unsigned)W);
      const int w = (int)(u - d * hw - h * (unsigned)W);
      m[0] = max(m[0], D - d); m[1] = max(m[1], d + 1);
      m[2] = max(m[2], H - h); m[3] = max(m[3], h + 1);
      m[4] = max(m[4], W - w); m[5] = max(m[5], w + 1);
    }
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const int r = fg_wmax(m[k]);
    if (lane == 0) red[k][wid] = r;
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    int r = 0;
    for (int i = 0; i < kFgThreads / 32; ++i) r = max(r, red[threadIdx.x][i]);
    if (r > 0) atomicMax(acc + n * 6 + threadIdx.x, r);
  }
}

// one thread per sample: box = [first - margin, last + margin + 1) per axis (MONAI generate_spatial_bounding_box), clipped to
// the volume when allow_smaller; an empty mask (or crop = 0) takes the whole volume.  Source index of output index p on the
// (OD, OH, OW) grid: b + s (A p) + (s - 1) / 2 with s = box size / output size (MONAI's lazy Resize, = interpolate(align_corners
// =False)), composed in fp64 and rounded to fp32 once.
__global__ void k_fg_compose(const AugSample* __restrict__ samples, int N, const int* __restrict__ acc, int margin, int allow_smaller,
                             const double* __restrict__ affine_in, int OD, int OH, int OW, float* __restrict__ affine_out,
                             int32_t* __restrict__ box, int32_t* __restrict__ empty) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const AugSample sm = samples[n];
  const int ext[3] = {(int)sm.d, (int)sm.h, (int)sm.w};
  const int out[3] = {OD, OH, OW};
  const bool none = acc == nullptr || acc[n * 6] == 0;
  for (int a = 0; a < 3; ++a) {
    int b0 = 0, b1 = ext[a];
    if (!none) {
      b0 = ext[a] - acc[n * 6 + 2 * a] - margin;
      b1 = acc[n * 6 + 2 * a + 1] + margin;
      if (allow_smaller) { b0 = max(b0, 0); b1 = min(b1, ext[a]); }
    }
    box[n * 6 + 2 * a] = b0;
    box[n * 6 + 2 * a + 1] = b1;
    const double s = (double)(b1 - b0) / (double)out[a];
    const double* m = affine_in + n * 12 + a * 4;
    float* o = affine_out + n * 12 + a * 4;
    for (int j = 0; j < 3; ++j) o[j] = (float)(s * m[j]);
    o[3] = (float)((double)b0 + s * m[3] + (s - 1.0) * 0.5);
  }
  empty[n] = acc != nullptr && acc[n * 6] == 0;
}

int launch_foreground_box(const AugSample* samples, int N, int C, long long max_spatial, int crop, const long long* ranks,
                          const float* gamma, int margin, int allow_smaller, const double* affine_in, int OD, int OH, int OW,
                          float* affine_out, int32_t* box, int32_t* empty, float* thr, void* scratch, cudaStream_t st) {
  B200_REQUIRE(samples && affine_in && affine_out && box && empty && scratch, E_INVALID, "foreground_box: null argument");
  B200_REQUIRE(!ranks || (gamma && thr), E_INVALID, "foreground_box: a percentile threshold needs gamma and thr");
  B200_REQUIRE(OD >= 1 && OH >= 1 && OW >= 1 && max_spatial >= 1 && max_spatial < (1LL << 31) && margin >= 0, E_INVALID,
               "foreground_box: bad output %dx%dx%d, largest sample %lld voxels, margin %d", OD, OH, OW, max_spatial, margin);
  const size_t bytes = foreground_scratch_bytes(N, C);
  if (bytes == 0) return E_UNSUPPORTED;
  const int P = N * C;
  unsigned* hist = reinterpret_cast<unsigned*>(scratch);
  FgPlane* planes = reinterpret_cast<FgPlane*>(reinterpret_cast<char*>(scratch) + fg_hist_bytes(P));
  int* acc = reinterpret_cast<int*>(planes + P);
  if (crop) {
    B200_CHECK_CUDA(cudaMemsetAsync(scratch, 0, bytes, st));
    auto blocks = [&](int rows) {
      long long b = (max_spatial + kFgThreads * kFgUnroll * 8 - 1) / (kFgThreads * kFgUnroll * 8);
      const long long cap = (kFgTargetBlocks + rows - 1) / rows;
      return (unsigned)(b < 1 ? 1 : b > cap ? cap : b);
    };
    if (ranks) {
      for (int pass = 0; pass < 3; ++pass) {
        k_fg_hist<<<dim3(blocks(P), P), kFgThreads, 0, st>>>(samples, C, pass, planes, hist);
        B200_CHECK_CUDA(cudaGetLastError());
        k_fg_scan<<<P, kFgThreads, 0, st>>>(pass, ranks, gamma, planes, hist, thr);
        B200_CHECK_CUDA(cudaGetLastError());
      }
    }
    k_fg_box<<<dim3(blocks(N), N), kFgThreads, 0, st>>>(samples, C, ranks ? thr : nullptr, acc);
    B200_CHECK_CUDA(cudaGetLastError());
  }
  k_fg_compose<<<(N + 127) / 128, 128, 0, st>>>(samples, N, crop ? acc : nullptr, margin, allow_smaller, affine_in, OD, OH, OW,
                                                affine_out, box, empty);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

}  // namespace b200
