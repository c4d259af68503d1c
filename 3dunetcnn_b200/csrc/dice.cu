// Per-voxel sigmoid-Dice criterion, forward and backward (HBM-bound reductions).
//
// Restates monai.losses.DiceLoss as selected by the reference's JSON config
// (/root/reference/unet3d/scripts/script_utils.py:61-77, examples/brats2020/brats2020_config.json:112-116):
//   p = sigmoid(x);  per (n,c):  I = sum p*t,  P = sum p (or p^2),  T = sum t (or t^2)
//   f = 1 - (2I + nr) / (P + T + dr)      [jaccard: denominator 2*(P + T - I)]
//   loss = mean_{n,c} f                   [batch=True: sums are pooled over n first]
// logits are NCDHW fp32, targets uint8 one-hot (unet3d/transforms/one_hot.py:10) - read as stored, no casts in HBM - or
// fp32 (soft / interpolated / label-smoothed targets, which MONAI accepts: flag bit 6).
#include "kernels.h"

namespace b200 {

struct DiceFlags {
  int sigmoid, squared_pred, jaccard, batch, include_background, reduction;  // reduction: 0 mean, 1 sum
};

__device__ __forceinline__ float dice_prob(float x, int sigmoid) { return sigmoid ? 1.f / (1.f + __expf(-x)) : x; }

__device__ __forceinline__ double block_sum(double v, double* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) sh[w] = v;
  __syncthreads();
  double r = 0;
  if (threadIdx.x < 32) {
    r = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  }
  __syncthreads();
  return r;
}

// grid (chunks, N*C); sums[(n*C+c)*3 + {0,1,2}] += (I, P, T).  vec: 4 voxels per load (uint8 targets only; the launcher
// checks S % 4 and the alignment of both pointers)
template <typename TT>
__global__ void k_dice_sums(const float* __restrict__ x, const TT* __restrict__ t, long long S, int vec, DiceFlags f,
                            double* __restrict__ sums) {
  __shared__ double sh[32];
  const long long base = (long long)blockIdx.y * S;
  float aI = 0.f, aP = 0.f, aT = 0.f;
  if (vec && sizeof(TT) == 1) {
    const float4* x4 = reinterpret_cast<const float4*>(x + base);
    const uchar4* t4 = reinterpret_cast<const uchar4*>(t + base);
    const long long n4 = S >> 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
      const float4 xv = __ldg(x4 + i);
      const uchar4 tv = __ldg(t4 + i);
      const float p0 = dice_prob(xv.x, f.sigmoid), p1 = dice_prob(xv.y, f.sigmoid), p2 = dice_prob(xv.z, f.sigmoid),
                  p3 = dice_prob(xv.w, f.sigmoid);
      const float t0 = tv.x, t1 = tv.y, t2 = tv.z, t3 = tv.w;
      aI += p0 * t0 + p1 * t1 + p2 * t2 + p3 * t3;
      if (f.squared_pred) {
        aP += p0 * p0 + p1 * p1 + p2 * p2 + p3 * p3;
        aT += t0 * t0 + t1 * t1 + t2 * t2 + t3 * t3;
      } else {
        aP += p0 + p1 + p2 + p3;
        aT += t0 + t1 + t2 + t3;
      }
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < S; i += (long long)gridDim.x * blockDim.x) {
      const float p = dice_prob(x[base + i], f.sigmoid);
      const float tt = t[base + i];
      aI += p * tt;
      aP += f.squared_pred ? p * p : p;
      aT += f.squared_pred ? tt * tt : tt;
    }
  }
  const double rI = block_sum((double)aI, sh), rP = block_sum((double)aP, sh), rT = block_sum((double)aT, sh);
  if (threadIdx.x == 0) {
    atomicAdd(&sums[(long long)blockIdx.y * 3 + 0], rI);
    atomicAdd(&sums[(long long)blockIdx.y * 3 + 1], rP);
    atomicAdd(&sums[(long long)blockIdx.y * 3 + 2], rT);
  }
}

__global__ void k_dice_finalize(const double* __restrict__ sums, int N, int C, DiceFlags f, float nr, float dr,
                                float* __restrict__ loss) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int c_lo = (!f.include_background && C > 1) ? 1 : 0;
  double acc = 0;
  int cnt = 0;
  if (f.batch) {
    for (int c = c_lo; c < C; ++c) {
      double I = 0, P = 0, T = 0;
      for (int n = 0; n < N; ++n) { I += sums[(n * C + c) * 3]; P += sums[(n * C + c) * 3 + 1]; T += sums[(n * C + c) * 3 + 2]; }
      double den = P + T;
      if (f.jaccard) den = 2.0 * (den - I);
      acc += 1.0 - (2.0 * I + nr) / (den + dr);
      ++cnt;
    }
  } else {
    for (int n = 0; n < N; ++n)
      for (int c = c_lo; c < C; ++c) {
        const double I = sums[(n * C + c) * 3], P = sums[(n * C + c) * 3 + 1], T = sums[(n * C + c) * 3 + 2];
        double den = P + T;
        if (f.jaccard) den = 2.0 * (den - I);
        acc += 1.0 - (2.0 * I + nr) / (den + dr);
        ++cnt;
      }
  }
  *loss = (float)(f.reduction == 0 ? acc / cnt : acc);
}

// dL/dx = g * w_nc * [ dF/dI * t + dF/dP * dP/dp ] * p(1-p)
//   F = 1 - (2I+nr)/(Den+dr);  plain: Den = P+T  ->  dF/dI = -2/D', dF/dP = (2I+nr)/D'^2
//   jaccard: Den = 2(P+T-I)    ->  dF/dI = -2/D' - 2(2I+nr)/D'^2 , dF/dP = 2(2I+nr)/D'^2          (D' = Den + dr)
template <typename TT>
__global__ void k_dice_bwd(const float* __restrict__ x, const TT* __restrict__ t, int N, int C, long long S,
                           DiceFlags f, float nr, float dr, const double* __restrict__ sums,
                           const float* __restrict__ grad_out, float* __restrict__ dx) {
  const int nc = blockIdx.y;
  const int n = nc / C, c = nc % C;
  const int c_lo = (!f.include_background && C > 1) ? 1 : 0;
  double I = 0, P = 0, T = 0;
  if (f.batch) {
    for (int m = 0; m < N; ++m) { I += sums[(m * C + c) * 3]; P += sums[(m * C + c) * 3 + 1]; T += sums[(m * C + c) * 3 + 2]; }
  } else {
    I = sums[(n * C + c) * 3]; P = sums[(n * C + c) * 3 + 1]; T = sums[(n * C + c) * 3 + 2];
  }
  double den = P + T;
  if (f.jaccard) den = 2.0 * (den - I);
  const double D = den + dr;
  const double num = 2.0 * I + nr;
  double dFdI = -2.0 / D, dFdP = num / (D * D);
  if (f.jaccard) { dFdI = -2.0 / D - 2.0 * num / (D * D); dFdP = 2.0 * num / (D * D); }
  const int terms = f.batch ? (C - c_lo) : N * (C - c_lo);
  double wgt = (f.reduction == 0 ? 1.0 / terms : 1.0) * (double)(*grad_out);
  if (c < c_lo) wgt = 0.0;
  const float a = (float)(wgt * dFdI), b = (float)(wgt * dFdP);
  const long long base = (long long)nc * S;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < S; i += (long long)gridDim.x * blockDim.x) {
    const float xv = x[base + i];
    const float p = dice_prob(xv, f.sigmoid);
    const float tt = t[base + i];
    const float dp = f.sigmoid ? p * (1.f - p) : 1.f;
    const float dPdp = f.squared_pred ? 2.f * p : 1.f;
    dx[base + i] = (a * tt + b * dPdp) * dp;
  }
}

static DiceFlags unpack_flags(int flags) {
  DiceFlags f;
  f.sigmoid = flags & 1; f.squared_pred = (flags >> 1) & 1; f.jaccard = (flags >> 2) & 1; f.batch = (flags >> 3) & 1;
  f.include_background = !((flags >> 4) & 1);
  f.reduction = (flags >> 5) & 1;
  return f;
}

int launch_dice_fwd(const float* logits, const uint8_t* target, int N, int C, long long S, int flags, float nr,
                    float dr, double* sums, float* loss, cudaStream_t st) {
  B200_REQUIRE(N > 0 && C > 0 && S > 0, E_INVALID, "dice: empty input");
  DiceFlags f = unpack_flags(flags);
  B200_CHECK_CUDA(cudaMemsetAsync(sums, 0, sizeof(double) * 3 * N * C, st));
  long long per = (S + 1023) / 1024;
  int chunks = (int)(per < 1 ? 1 : per);
  int cap = (132 * 8 + N * C - 1) / (N * C);
  if (chunks > cap) chunks = cap < 1 ? 1 : cap;
  // float4 / uchar4 loads need S % 4 == 0 and 16- / 4-byte aligned pointers: a contiguous view at a storage offset (a slice
  // of a wider tensor) may not be, and takes the scalar loop
  const int vec = (S & 3) == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0 && (reinterpret_cast<uintptr_t>(target) & 3) == 0;
  if (flags & 64)
    k_dice_sums<float><<<dim3(chunks, N * C), 256, 0, st>>>(logits, reinterpret_cast<const float*>(target), S, 0, f, sums);
  else k_dice_sums<uint8_t><<<dim3(chunks, N * C), 256, 0, st>>>(logits, target, S, vec, f, sums);
  B200_CHECK_CUDA(cudaGetLastError());
  k_dice_finalize<<<1, 32, 0, st>>>(sums, N, C, f, nr, dr, loss);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

int launch_dice_bwd(const float* logits, const uint8_t* target, int N, int C, long long S, int flags, float nr,
                    float dr, const double* sums, const float* grad_out, float* dlogits, cudaStream_t st) {
  DiceFlags f = unpack_flags(flags);
  long long per = (S + 1023) / 1024;
  int chunks = (int)(per < 1 ? 1 : per);
  int cap = (132 * 8 + N * C - 1) / (N * C);
  if (chunks > cap) chunks = cap < 1 ? 1 : cap;
  if (flags & 64)
    k_dice_bwd<float><<<dim3(chunks, N * C), 256, 0, st>>>(logits, reinterpret_cast<const float*>(target), N, C, S, f, nr, dr, sums,
                                                            grad_out, dlogits);
  else k_dice_bwd<uint8_t><<<dim3(chunks, N * C), 256, 0, st>>>(logits, target, N, C, S, f, nr, dr, sums, grad_out, dlogits);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

}  // namespace b200
