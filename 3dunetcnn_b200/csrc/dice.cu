// Dice criterion: the one finalize (loss and backward coefficients) of both Dice criteria, and DiceLoss's own per-voxel
// sums and backward (HBM-bound reductions).
//
// Restates monai.losses.DiceLoss as selected by the reference's JSON config
// (/root/reference/unet3d/scripts/script_utils.py:61-77, examples/brats2020/brats2020_config.json:112-116):
//   p = sigmoid(x) or x;  per (n,c):  I = sum p*t,  P = sum p (or p^2),  T = sum t (or t^2)
//   f = 1 - (2I + nr) / (P + T + dr)      [jaccard: denominator 2*(P + T - I)]
//   loss = lambda_dice * mean_{n,c} f     [batch=True: sums are pooled over n first]
// DiceLoss: logits are NCDHW fp32, targets uint8 one-hot (unet3d/transforms/one_hot.py:10) - read as stored, no casts in
// HBM - or fp32 (soft / interpolated / label-smoothed targets, which MONAI accepts).  Its options are a DiceCEDesc with no
// softmax, a C-channel target and lambda_ce = 0; dice_ce.cu runs the rest on its staged-tile kernels.
#include "kernels.h"

namespace b200 {

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
__global__ void k_dice_sums(const float* __restrict__ x, const TT* __restrict__ t, long long S, int vec, DiceCEDesc d,
                            double* __restrict__ sums) {
  __shared__ double sh[32];
  const long long base = (long long)blockIdx.y * S;
  const int sig = d.act == A_SIGMOID;
  float aI = 0.f, aP = 0.f, aT = 0.f;
  if (vec && sizeof(TT) == 1) {
    const float4* x4 = reinterpret_cast<const float4*>(x + base);
    const uchar4* t4 = reinterpret_cast<const uchar4*>(t + base);
    const long long n4 = S >> 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
      const float4 xv = __ldg(x4 + i);
      const uchar4 tv = __ldg(t4 + i);
      const float p0 = dice_prob(xv.x, sig), p1 = dice_prob(xv.y, sig), p2 = dice_prob(xv.z, sig), p3 = dice_prob(xv.w, sig);
      const float t0 = tv.x, t1 = tv.y, t2 = tv.z, t3 = tv.w;
      aI += p0 * t0 + p1 * t1 + p2 * t2 + p3 * t3;
      if (d.squared_pred) {
        aP += p0 * p0 + p1 * p1 + p2 * p2 + p3 * p3;
        aT += t0 * t0 + t1 * t1 + t2 * t2 + t3 * t3;
      } else {
        aP += p0 + p1 + p2 + p3;
        aT += t0 + t1 + t2 + t3;
      }
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < S; i += (long long)gridDim.x * blockDim.x) {
      const float p = dice_prob(x[base + i], sig);
      const float tt = t[base + i];
      aI += p * tt;
      aP += d.squared_pred ? p * p : p;
      aT += d.squared_pred ? tt * tt : tt;
    }
  }
  const double rI = block_sum((double)aI, sh), rP = block_sum((double)aP, sh), rT = block_sum((double)aT, sh);
  if (threadIdx.x == 0) {
    atomicAdd(&sums[(long long)blockIdx.y * 3 + 0], rI);
    atomicAdd(&sums[(long long)blockIdx.y * 3 + 1], rP);
    atomicAdd(&sums[(long long)blockIdx.y * 3 + 2], rT);
  }
}

__device__ __forceinline__ void pooled(const double* sums, int N, int C, int n, int c, int batch, double& I, double& P, double& T) {
  if (batch) {
    I = P = T = 0;
    for (int m = 0; m < N; ++m) { I += sums[(m * C + c) * 3]; P += sums[(m * C + c) * 3 + 1]; T += sums[(m * C + c) * 3 + 2]; }
  } else {
    I = sums[(n * C + c) * 3]; P = sums[(n * C + c) * 3 + 1]; T = sums[(n * C + c) * 3 + 2];
  }
}

// f of one (n, c) pair (Dice, Jaccard or Tversky) and its (dF/dI, dF/dP):
//   F = 1 - (2I+nr)/(Den+dr);  plain: Den = P+T  ->  dF/dI = -2/D', dF/dP = (2I+nr)/D'^2
//   jaccard: Den = 2(P+T-I)    ->  dF/dI = -2/D' - 2(2I+nr)/D'^2 , dF/dP = 2(2I+nr)/D'^2          (D' = Den + dr)
//   Tversky: F = 1 - (I+nr)/D', D' = I + a(P-I) + b(T-I) + dr  ->  dF/dI = -1/D' + (I+nr)(1-a-b)/D'^2, dF/dP = a(I+nr)/D'^2
__device__ __forceinline__ double overlap_f(const DiceCEDesc& d, double I, double P, double T, double& dFdI, double& dFdP) {
  if (d.overlap == O_TVERSKY) {
    const double a = d.tversky_alpha, b = d.tversky_beta;
    const double D = I + a * (P - I) + b * (T - I) + d.smooth_dr, num = I + d.smooth_nr;
    dFdI = -1.0 / D + num * (1.0 - a - b) / (D * D);
    dFdP = a * num / (D * D);
    return 1.0 - num / D;
  }
  double den = P + T;
  if (d.jaccard) den = 2.0 * (den - I);
  const double D = den + d.smooth_dr, num = 2.0 * I + d.smooth_nr;
  dFdI = -2.0 / D; dFdP = num / (D * D);
  if (d.jaccard) { dFdI = -2.0 / D - 2.0 * num / (D * D); dFdP = 2.0 * num / (D * D); }
  return 1.0 - (2.0 * I + d.smooth_nr) / (den + d.smooth_dr);
}

// generalized Dice weight of a class with target sum T (inf when T == 0 and the weight is not uniform)
__device__ __forceinline__ double gdice_weight(double T, int w_type) {
  return w_type == W_SQUARE ? 1.0 / (T * T) : w_type == W_SIMPLE ? 1.0 / T : 1.0;
}

// Generalized Dice of group g (sample g, or every sample with batch): the largest finite weight, which replaces the infinite
// ones, and A = 2 sum_c w_c I_c + nr, B = sum_c w_c (P_c + T_c) + dr over the kept channels
__device__ void gdice_group(const double* sums, int N, int C, int g, int c_lo, const DiceCEDesc& d, double* out) {
  double wmax = 0;
  for (int c = c_lo; c < C; ++c) {
    double I, P, T;
    pooled(sums, N, C, g, c, d.batch, I, P, T);
    const double w = gdice_weight(T, d.w_type);
    if (!isinf(w)) wmax = fmax(wmax, w);
  }
  double A = 0, B = 0;
  for (int c = c_lo; c < C; ++c) {
    double I, P, T;
    pooled(sums, N, C, g, c, d.batch, I, P, T);
    double w = gdice_weight(T, d.w_type);
    if (isinf(w)) w = wmax;
    A += w * I;
    B += w * (P + T);
  }
  out[0] = 2.0 * A + d.smooth_nr;
  out[1] = B + d.smooth_dr;
  out[2] = wmax;
}

// coef [N][C][2] = lambda_dice * w * (dF/dI, dF/dP), zero on a dropped background channel and everywhere when lambda_dice = 0;
// the scalar loss.  The backward kernels form dL/dx = g * [ coef_I * t + coef_P * dP/dp ] * dp/dx.  ce [N] is read only when
// lambda_ce != 0.  Generalized Dice couples a group's classes through A and B: f = 1 - A/B, dF/dI_c = -2 w_c / B,
// dF/dP_c = A w_c / B^2; the groups are formed 128 at a time, then their pairs' coefficients.
__global__ void k_dice_finalize(const double* __restrict__ sums, const double* __restrict__ ce, int N, int C, long long S, DiceCEDesc d,
                                double* __restrict__ coef, float* __restrict__ loss) {
  const int c_lo = (!d.include_background && C > 1) ? 1 : 0;
  double acc = 0;
  if (d.lambda_dice == 0.f) {
    for (int i = threadIdx.x; i < N * C; i += blockDim.x) coef[i * 2] = coef[i * 2 + 1] = 0.0;
  } else if (d.overlap == O_GDICE) {
    __shared__ double grp[128][3];
    const int G = d.batch ? 1 : N;
    const double w = d.lambda_dice * (d.reduction == 0 ? 1.0 / G : 1.0);
    for (int g0 = 0; g0 < G; g0 += 128) {
      const int ng = min(128, G - g0);
      if ((int)threadIdx.x < ng) gdice_group(sums, N, C, g0 + threadIdx.x, c_lo, d, grp[threadIdx.x]);
      __syncthreads();
      const int n0 = d.batch ? 0 : g0, rows = d.batch ? N : ng;
      for (int i = threadIdx.x; i < rows * C; i += blockDim.x) {
        const int n = n0 + i / C, c = i % C;
        const double* q = grp[d.batch ? 0 : n - g0];
        double I, P, T;
        pooled(sums, N, C, n, c, d.batch, I, P, T);
        double wc = gdice_weight(T, d.w_type);
        if (isinf(wc)) wc = q[2];
        if (c < c_lo) wc = 0.0;
        coef[((long long)n * C + c) * 2] = w * (-2.0 * wc / q[1]);
        coef[((long long)n * C + c) * 2 + 1] = w * (q[0] * wc / (q[1] * q[1]));
      }
      if (threadIdx.x == 0)
        for (int g = 0; g < ng; ++g) acc += 1.0 - grp[g][0] / grp[g][1];
      __syncthreads();
    }
    if (threadIdx.x != 0) return;
    acc = d.lambda_dice * (d.reduction == 0 ? acc / G : acc);
  } else {
    const int terms = (d.batch ? 1 : N) * (C - c_lo);
    const double w = d.lambda_dice * (d.reduction == 0 ? 1.0 / terms : 1.0);
    for (int i = threadIdx.x; i < N * C; i += blockDim.x) {
      const int n = i / C, c = i % C;
      double I, P, T, dFdI, dFdP;
      pooled(sums, N, C, n, c, d.batch, I, P, T);
      overlap_f(d, I, P, T, dFdI, dFdP);
      const double wc = c < c_lo ? 0.0 : w;
      coef[i * 2] = wc * dFdI;
      coef[i * 2 + 1] = wc * dFdP;
    }
    if (threadIdx.x != 0) return;
    for (int n = 0; n < (d.batch ? 1 : N); ++n)
      for (int c = c_lo; c < C; ++c) {
        double I, P, T, dFdI, dFdP;
        pooled(sums, N, C, n, c, d.batch, I, P, T);
        acc += overlap_f(d, I, P, T, dFdI, dFdP);
      }
    acc = d.lambda_dice * (d.reduction == 0 ? acc / terms : acc);
  }
  if (threadIdx.x != 0) return;
  double l = acc;
  if (d.lambda_ce != 0.f) {
    double cet = 0;
    for (int n = 0; n < N; ++n) cet += ce[n];
    l += d.lambda_ce * (cet / voxel_divisor(d, N, C, S));
  }
  *loss = (float)l;
}

// grid (chunks, N*C); (a, b) = coef of this (n, c) times grad_out, so the voxel loop does only fp32 work
template <typename TT>
__global__ void k_dice_bwd(const float* __restrict__ x, const TT* __restrict__ t, long long S, DiceCEDesc d,
                           const double* __restrict__ coef, const float* __restrict__ grad_out, float* __restrict__ dx) {
  const int nc = blockIdx.y;
  const int sig = d.act == A_SIGMOID;
  const float go = *grad_out;
  const float a = (float)(coef[nc * 2] * go), b = (float)(coef[nc * 2 + 1] * go);
  const long long base = (long long)nc * S;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < S; i += (long long)gridDim.x * blockDim.x) {
    const float xv = x[base + i];
    const float p = dice_prob(xv, sig);
    const float tt = t[base + i];
    const float dp = sig ? p * (1.f - p) : 1.f;
    const float dPdp = d.squared_pred ? 2.f * p : 1.f;
    dx[base + i] = (a * tt + b * dPdp) * dp;
  }
}

int check_dice_desc(const DiceCEDesc& d, int N, int C, long long S, const char* who) {
  B200_REQUIRE(N > 0 && C > 0 && S > 0, E_INVALID, "%s: empty input (n=%d c=%d spatial=%lld)", who, N, C, S);
  B200_REQUIRE(d.act >= 0 && d.act <= 2, E_INVALID, "%s: act=%d (0 none, 1 sigmoid, 2 softmax)", who, d.act);
  B200_REQUIRE(d.target_kind >= 0 && d.target_kind <= 3, E_INVALID, "%s: target_kind=%d", who, d.target_kind);
  B200_REQUIRE(d.reduction == 0 || d.reduction == 1, E_INVALID, "%s: reduction=%d (0 mean, 1 sum)", who, d.reduction);
  B200_REQUIRE(d.lambda_dice >= 0.f && d.lambda_ce >= 0.f, E_INVALID, "%s: negative lambda", who);
  B200_REQUIRE(d.overlap >= 0 && d.overlap <= 2, E_INVALID, "%s: overlap=%d (0 Dice, 1 Tversky, 2 generalized Dice)", who, d.overlap);
  B200_REQUIRE(d.overlap == O_DICE || (!d.squared_pred && !d.jaccard), E_INVALID,
               "%s: squared_pred / jaccard apply to the Dice overlap only (overlap=%d)", who, d.overlap);
  B200_REQUIRE(d.w_type >= 0 && d.w_type <= 2, E_INVALID, "%s: w_type=%d (0 square, 1 simple, 2 uniform)", who, d.w_type);
  B200_REQUIRE(d.voxel_term >= V_CE && d.voxel_term <= V_HDT, E_INVALID, "%s: voxel_term=%d (0 CE, 1 focal, 2 distance-weighted)", who,
               d.voxel_term);
  B200_REQUIRE(d.focal_gamma >= 0.f, E_INVALID, "%s: focal_gamma=%g (>= 0)", who, d.focal_gamma);
  return OK;
}

int launch_dice_finalize(const DiceCEDesc& d, const double* sums, const double* ce, int N, int C, long long S, double* coef,
                         float* loss, cudaStream_t st) {
  k_dice_finalize<<<1, 128, 0, st>>>(sums, ce, N, C, S, d, coef, loss);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

static int check_dice(const DiceCEDesc& d, int N, int C, long long S) {
  B200_TRY(check_dice_desc(d, N, C, S, "dice"));
  B200_REQUIRE(d.act != A_SOFTMAX, E_UNSUPPORTED, "dice: softmax is not implemented here (b200unet_dice_ce_* runs it)");
  B200_REQUIRE(d.target_kind == T_ONEHOT_U8 || d.target_kind == T_SOFT_F32, E_UNSUPPORTED,
               "dice: target_kind=%d (a label map goes to b200unet_dice_ce_*; here 2 uint8 or 3 fp32 [n][c][spatial])", d.target_kind);
  B200_REQUIRE(d.lambda_ce == 0.f, E_INVALID, "dice: lambda_ce=%g (the CE term is computed by b200unet_dice_ce_*)", d.lambda_ce);
  B200_REQUIRE(d.overlap == O_DICE && d.voxel_term == V_CE && !d.focal_softmax && !d.focal_use_alpha && !d.class_weight,
               E_UNSUPPORTED, "dice: overlap=%d voxel_term=%d (Tversky, generalized Dice and the focal term run on b200unet_dice_ce_*)",
               d.overlap, d.voxel_term);
  return OK;
}

// chunks per (n, c): one per 1024 voxels, at most 8 blocks per SM over the N*C rows of the 132-SM grid
static int dice_chunks(int N, int C, long long S) {
  long long per = (S + 1023) / 1024;
  int chunks = (int)(per < 1 ? 1 : per);
  int cap = (132 * 8 + N * C - 1) / (N * C);
  if (chunks > cap) chunks = cap < 1 ? 1 : cap;
  return chunks;
}

int launch_dice_fwd(const DiceCEDesc& d, const float* logits, const void* target, int N, int C, long long S, double* scratch,
                    float* loss, cudaStream_t st) {
  B200_TRY(check_dice(d, N, C, S));
  double* sums = scratch;
  B200_CHECK_CUDA(cudaMemsetAsync(sums, 0, sizeof(double) * 3 * N * C, st));
  const int chunks = dice_chunks(N, C, S);
  // float4 / uchar4 loads need S % 4 == 0 and 16- / 4-byte aligned pointers: a contiguous view at a storage offset (a slice
  // of a wider tensor) may not be, and takes the scalar loop
  const int vec = (S & 3) == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0 && (reinterpret_cast<uintptr_t>(target) & 3) == 0;
  if (d.target_kind == T_SOFT_F32)
    k_dice_sums<float><<<dim3(chunks, N * C), 256, 0, st>>>(logits, static_cast<const float*>(target), S, 0, d, sums);
  else k_dice_sums<uint8_t><<<dim3(chunks, N * C), 256, 0, st>>>(logits, static_cast<const uint8_t*>(target), S, vec, d, sums);
  B200_CHECK_CUDA(cudaGetLastError());
  return launch_dice_finalize(d, sums, nullptr, N, C, S, sums + (size_t)N * C * 3, loss, st);
}

int launch_dice_bwd(const DiceCEDesc& d, const float* logits, const void* target, int N, int C, long long S, const double* scratch,
                    const float* grad_out, float* dlogits, cudaStream_t st) {
  B200_TRY(check_dice(d, N, C, S));
  const double* coef = scratch + (size_t)N * C * 3;
  const int chunks = dice_chunks(N, C, S);
  if (d.target_kind == T_SOFT_F32)
    k_dice_bwd<float><<<dim3(chunks, N * C), 256, 0, st>>>(logits, static_cast<const float*>(target), S, d, coef, grad_out, dlogits);
  else k_dice_bwd<uint8_t><<<dim3(chunks, N * C), 256, 0, st>>>(logits, static_cast<const uint8_t*>(target), S, d, coef, grad_out,
                                                                 dlogits);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

}  // namespace b200
