// Bandwidth-bound kernels of the U-Net path (everything that is not a tensor-core contraction):
// input packing, GroupNorm apply/backward, trilinear x2 up-sampling fwd/bwd, 1x1x1 head fwd/bwd
// and zero insertion (weight packing: small_ops.cu).  All activations are NDHWC bf16 (hi [+ lo]) views; 8 channels (16 B) per
// thread so every access is a 128-bit vector along the innermost (channel) axis.
//
// Reference semantics restated (paths relative to /root/reference):
//   GroupNorm+ReLU      unet3d/models/pytorch/classification/myronenko.py:17-31
//   trilinear x2        unet3d/models/pytorch/classification/decoder.py:105-106
//   final 1x1x1 conv    unet3d/models/pytorch/autoencoder/variational.py:59-60,84
#include "kernels.h"
#include "ptx.cuh"

namespace b200 {

// ------------------------------------------------------------------------------------------------ helpers
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------ input pack
// x: NCDHW fp32 -> out: NDHWC bf16 (C padded with zeros to out.C), + per-(n,c) sum / sum-of-squares (double).
__global__ void k_input_pack(const float* __restrict__ x, int C, long long S, Act out, double* __restrict__ stats,
                             int stats_ld) {
  const int n = blockIdx.y;
  const int Cp = out.C;  // 8 or 16
  __shared__ double s_sum[16][2];   // fp64: the order of the per-warp atomics must not show in the fp32 coefficients
  if (threadIdx.x < 32) (&s_sum[0][0])[threadIdx.x] = 0.0;
  __syncthreads();
  float acc[16][2];
#pragma unroll
  for (int c = 0; c < 16; ++c) acc[c][0] = acc[c][1] = 0.f;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (long long)gridDim.x * blockDim.x) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h * 8 < Cp) {
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = h * 8 + j;
          v[j] = c < C ? x[((long long)n * C + c) * S + s] : 0.f;
          acc[h * 8 + j][0] += v[j];
          acc[h * 8 + j][1] += v[j] * v[j];
        }
        store8(out.hi, out.lo, ((long long)n * S + s) * out.ld + h * 8, v);
      }
    }
  }
  if (stats) {
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      if (c < C) {
        float a = warp_sum(acc[c][0]), b = warp_sum(acc[c][1]);
        if ((threadIdx.x & 31) == 0) { atomicAdd(&s_sum[c][0], (double)a); atomicAdd(&s_sum[c][1], (double)b); }
      }
    }
    __syncthreads();
    if (threadIdx.x < C) {
      atomicAdd(&stats[((long long)n * stats_ld + threadIdx.x) * 2 + 0], s_sum[threadIdx.x][0]);
      atomicAdd(&stats[((long long)n * stats_ld + threadIdx.x) * 2 + 1], s_sum[threadIdx.x][1]);
    }
  }
}

int launch_input_pack(const float* x, int C, const Act& out, double* stats, int stats_ld, cudaStream_t st) {
  B200_REQUIRE(C <= 16, E_UNSUPPORTED, "input_pack: n_features=%d > 16 unsupported", C);
  B200_REQUIRE(out.C % 8 == 0 && out.C >= C && out.C <= 16, E_INVALID, "input_pack: padded C=%d invalid", out.C);
  long long S = (long long)out.D * out.H * out.W;
  int threads = 256;
  int blocks = (int)((S + threads - 1) / threads);
  if (blocks > 1184) blocks = 1184;
  k_input_pack<<<dim3(blocks, out.N), threads, 0, st>>>(x, C, S, out, stats, stats_ld);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// ------------------------------------------------------------------------------------------------ GroupNorm apply (+ReLU / LeakyReLU)
// stats [N][x.C][2] (sum, sumsq over the S voxels of each of the C real channels) -> coef [N][x.C] = (A, B, mu, rstd):
//   z = A*x + B  with A = gamma*rstd, B = beta - mu*gamma*rstd ;  xhat = (x - mu)*rstd.    (biased variance, eps)
// y = act(z); padded channels (C <= c < x.C) get zero coefficients.
// grid (blocks, N); a thread keeps the same 8-channel chunk for its whole grid-stride loop (blockDim.x % c8n == 0),
// so the affine coefficients live in registers and the loop body is load -> 8 FMA/max -> store, two voxels in flight.
// Every block first derives the coefficients of its sample from the statistics (a few hundred fp64 loads, hidden behind
// the other resident blocks) instead of a separate single-block finalize launch per norm layer (~7 us each, 80 launches
// per step); block 0 of each sample also stores them for the backward pass.
struct GnFin {
  const double* stats; const float* gamma; const float* beta; int C; int G; double S; float eps; float4* coef_out;
};
__global__ void __launch_bounds__(256) k_gn_apply(Act x, Act y, float slope, GnFin f) {
  pdl_wait();                 // launched through launch_pdl: the producer of x / of the statistics has completed past this line
  pdl_launch_dependents();
  const int c8n = x.C / 8;
  const int n = blockIdx.y;
  const long long S = (long long)x.D * x.H * x.W;
  const int c8 = threadIdx.x % c8n;
  const int vslot = threadIdx.x / c8n;
  const int vper = blockDim.x / c8n;
  float ka[8], kb[8];
  // one global fp64 load pair per thread, the group sums then come from shared memory (a per-thread loop over the
  // group's channels in global memory serialised up to 64 L2 latencies in front of every block)
  __shared__ float2 s_ab[1024];
  __shared__ double s_st[1024][2];
  for (int c = threadIdx.x; c < x.C; c += blockDim.x) {
    s_st[c][0] = c < f.C ? f.stats[((long long)n * x.C + c) * 2 + 0] : 0.0;
    s_st[c][1] = c < f.C ? f.stats[((long long)n * x.C + c) * 2 + 1] : 0.0;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < x.C; c += blockDim.x) {
    float4 k = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < f.C) {
      const int cg = f.C / f.G, g = c / cg;
      double sm_ = 0, q = 0;
      for (int j = 0; j < cg; ++j) { sm_ += s_st[g * cg + j][0]; q += s_st[g * cg + j][1]; }
      const double m = f.S * cg;
      const double mu = sm_ / m;
      double var = q / m - mu * mu;
      if (var < 0) var = 0;
      const double rstd = 1.0 / sqrt(var + (double)f.eps);
      const double ga = f.gamma ? (double)f.gamma[c] : 1.0, be = f.beta ? (double)f.beta[c] : 0.0;
      k = make_float4((float)(ga * rstd), (float)(be - mu * ga * rstd), (float)mu, (float)rstd);
    }
    s_ab[c] = make_float2(k.x, k.y);
    if (blockIdx.x == 0) f.coef_out[(long long)n * x.C + c] = k;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 8; ++j) { ka[j] = s_ab[c8 * 8 + j].x; kb[j] = s_ab[c8 * 8 + j].y; }
  const long long base = (long long)n * S;
  const long long stride = (long long)gridDim.x * vper;
  long long s = (long long)blockIdx.x * vper + vslot;
  for (; s + stride < S; s += 2 * stride) {
    float v0[8], v1[8];
    load8(x.hi, x.lo, (base + s) * x.ld + c8 * 8, v0);
    load8(x.hi, x.lo, (base + s + stride) * x.ld + c8 * 8, v1);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float z0 = fmaf(ka[j], v0[j], kb[j]), z1 = fmaf(ka[j], v1[j], kb[j]);
      v0[j] = z0 > 0.f ? z0 : z0 * slope;
      v1[j] = z1 > 0.f ? z1 : z1 * slope;
    }
    store8(y.hi, y.lo, (base + s) * y.ld + c8 * 8, v0);
    store8(y.hi, y.lo, (base + s + stride) * y.ld + c8 * 8, v1);
  }
  if (s < S) {
    float v0[8];
    load8(x.hi, x.lo, (base + s) * x.ld + c8 * 8, v0);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float z0 = fmaf(ka[j], v0[j], kb[j]);
      v0[j] = z0 > 0.f ? z0 : z0 * slope;
    }
    store8(y.hi, y.lo, (base + s) * y.ld + c8 * 8, v0);
  }
}

static int ew_blocks(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  long long cap = 132LL * 16;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

// threads per block: a multiple of c8n, at most 256 (the kernels' launch bound), a multiple of 32 when one exists
static int ew_threads_for(int c8n) {
  for (int t = 256; t >= 32; t -= 32)
    if (t % c8n == 0) return t;
  return c8n <= 256 ? (256 / c8n) * c8n : c8n;
}

// block size and grid of k_gn_apply / k_gn_bwd (x.C <= 1024, so threads <= 256): two voxels per thread per grid step, at
// most 8 blocks per SM over the whole batch
static void gn_launch_dims(const Act& x, dim3& grid, dim3& block) {
  const int c8n = x.C / 8;
  const int threads = ew_threads_for(c8n);
  const long long S = (long long)x.D * x.H * x.W;
  const int vper = threads / c8n;
  long long want = (S + 2LL * vper - 1) / (2LL * vper);
  const long long cap = (132LL * 8 + x.N - 1) / x.N;
  grid = dim3((int)(want < cap ? (want > 0 ? want : 1) : cap), x.N);
  block = dim3(threads);
}

// statistics -> coefficients -> y = act(A x + B) in one launch; coef [N][x.C] float4 is written for the backward pass
int launch_gn_apply(const Act& x, const Act& y, const double* stats, const float* gamma, const float* beta, int C, int G,
                    long long S, float eps, float* coef, float slope, cudaStream_t st) {
  B200_REQUIRE(x.C % 8 == 0 && y.C == x.C, E_INVALID, "gn_apply: C=%d/%d", x.C, y.C);
  B200_REQUIRE(G > 0 && C % G == 0 && C <= x.C, E_INVALID, "gn_apply: C=%d G=%d", C, G);
  B200_REQUIRE(x.C <= 1024, E_UNSUPPORTED, "gn_apply: C <= 1024 supported (got %d)", x.C);
  GnFin f;
  f.stats = stats; f.gamma = gamma; f.beta = beta; f.C = C; f.G = G; f.S = (double)S; f.eps = eps;
  f.coef_out = reinterpret_cast<float4*>(coef);
  dim3 grid, block;
  gn_launch_dims(x, grid, block);
  launch_pdl(k_gn_apply, grid, block, 0, st, x, y, slope, f);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// ------------------------------------------------------------------------------------------------ GroupNorm backward
// bstats [N][C][2] = (S1 = sum dz, S2 = sum dz*xhat) per (n,c);   dz = dL/dz (already ReLU-masked).
// coef2 [N][C][2] = (E, F):   dx = A*dz + E*x + F      (A from coef)
//   c1_g = (1/m) sum_{c in g} gamma_c S1_c ; c2_g = (1/m) sum gamma_c S2_c ; E = -rstd^2 c2 ; F = -rstd c1 + rstd^2 c2 mu
// dgamma_c = sum_n S2 ; dbeta_c = sum_n S1   (written, not accumulated)
// (E, F) of a channel from its group's gamma-weighted means c1 = sum gamma S1 / m, c2 = sum gamma S2 / m (m = S * cg values)
// and the channel's forward coefficients k = (A, B, mu, rstd)
__device__ __forceinline__ float2 gn_bwd_ef(double c1, double c2, float4 k) {
  const double mu = k.z, rstd = k.w;
  return make_float2((float)(-rstd * rstd * c2), (float)(-rstd * c1 + rstd * rstd * c2 * mu));
}

__global__ void k_gn_bwd_finalize(const double* __restrict__ bstats, const float4* __restrict__ coef,
                                  const float* __restrict__ gamma, int N, int C, int Cld, int G, double S,
                                  float2* __restrict__ coef2, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int cg = C / G;
  for (int c = threadIdx.x; c < Cld; c += blockDim.x) {
    if (c >= C) {
      for (int n = 0; n < N; ++n) coef2[(long long)n * Cld + c] = make_float2(0.f, 0.f);
      continue;
    }
    const int g = c / cg;
    double dg = 0, db = 0;
    for (int n = 0; n < N; ++n) {
      double c1 = 0, c2 = 0;
      for (int j = 0; j < cg; ++j) {
        const int cc = g * cg + j;
        const double ga = gamma ? (double)gamma[cc] : 1.0;
        c1 += ga * bstats[((long long)n * Cld + cc) * 2 + 0];
        c2 += ga * bstats[((long long)n * Cld + cc) * 2 + 1];
      }
      const double m = S * cg;
      c1 /= m; c2 /= m;
      coef2[(long long)n * Cld + c] = gn_bwd_ef(c1, c2, coef[(long long)n * Cld + c]);
      db += bstats[((long long)n * Cld + c) * 2 + 0];
      dg += bstats[((long long)n * Cld + c) * 2 + 1];
    }
    if (dgamma) dgamma[c] = (float)dg;
    if (dbeta) dbeta[c] = (float)db;
  }
}

int launch_gn_bwd_finalize(const double* bstats, const float* coef, const float* gamma, int N, int C, int Cld, int G,
                           long long S, float* coef2, float* dgamma, float* dbeta, cudaStream_t st) {
  B200_REQUIRE(G > 0 && C % G == 0 && Cld >= C, E_INVALID, "gn_bwd_finalize: C=%d G=%d", C, G);
  k_gn_bwd_finalize<<<1, 256, 0, st>>>(bstats, reinterpret_cast<const float4*>(coef), gamma, N, C, Cld, G, (double)S,
                                      reinterpret_cast<float2*>(coef2), dgamma, dbeta);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// dx = (A*dz + E*x + F (+ add1) (+ add2)) [* scale]     grid (blocks, N), per-thread constant channel chunk
// The blocks derive (E, F) themselves from the backward statistics and block (0, 0) also writes dgamma / dbeta (see k_gn_apply).
struct GnBwdFin {
  const double* bstats; const float* gamma; int C; int G; int N; double S; float* dgamma; float* dbeta;
};
__global__ void __launch_bounds__(256) k_gn_bwd(Act dz, Act x, const float4* __restrict__ coef, Act add1, Act add2, Act dx,
                                                const float* __restrict__ scale, GnBwdFin f) {
  pdl_wait();                 // launched through launch_pdl
  pdl_launch_dependents();
  const int c8n = x.C / 8;
  const int n = blockIdx.y;
  const long long S = (long long)x.D * x.H * x.W;
  const int c8 = threadIdx.x % c8n;
  const int vslot = threadIdx.x / c8n;
  const int vper = blockDim.x / c8n;
  float ka[8], ke[8], kf[8], ks[8];
  __shared__ float2 s_ef[1024];
  __shared__ double s_bs[1024][2];   // gamma-weighted backward statistics of every channel of this sample
  for (int c = threadIdx.x; c < x.C; c += blockDim.x) {
    const double ga = (c < f.C && f.gamma) ? (double)f.gamma[c] : 1.0;
    s_bs[c][0] = c < f.C ? ga * f.bstats[((long long)n * x.C + c) * 2 + 0] : 0.0;
    s_bs[c][1] = c < f.C ? ga * f.bstats[((long long)n * x.C + c) * 2 + 1] : 0.0;
    if (blockIdx.x == 0 && n == 0 && c < f.C) {
      double dg = 0, db = 0;
      for (int nn = 0; nn < f.N; ++nn) {
        db += f.bstats[((long long)nn * x.C + c) * 2 + 0];
        dg += f.bstats[((long long)nn * x.C + c) * 2 + 1];
      }
      if (f.dgamma) f.dgamma[c] = (float)dg;
      if (f.dbeta) f.dbeta[c] = (float)db;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < x.C; c += blockDim.x) {
    float2 e = make_float2(0.f, 0.f);
    if (c < f.C) {
      const int cg = f.C / f.G, g = c / cg;
      double c1 = 0, c2 = 0;
      for (int j = 0; j < cg; ++j) { c1 += s_bs[g * cg + j][0]; c2 += s_bs[g * cg + j][1]; }
      const double m = f.S * cg;
      c1 /= m; c2 /= m;
      e = gn_bwd_ef(c1, c2, coef[(long long)n * x.C + c]);
    }
    s_ef[c] = e;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    ka[j] = __ldg(coef + (long long)n * x.C + c8 * 8 + j).x;
    ke[j] = s_ef[c8 * 8 + j].x; kf[j] = s_ef[c8 * 8 + j].y;
    ks[j] = scale ? __ldg(scale + (long long)n * x.C + c8 * 8 + j) : 1.f;
  }
  const long long base = (long long)n * S;
  const long long stride = (long long)gridDim.x * vper;
  // two voxels in flight per thread: three streams (dz, x, optional adds) per voxel left the single-voxel loop at ~55% of
  // the HBM rate
  auto one = [&](long long vox, const float (&g)[8], const float (&v)[8]) {
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = fmaf(ka[j], g[j], fmaf(ke[j], v[j], kf[j]));
    if (add1.hi) {
      float a[8];
      load8(add1.hi, add1.lo, vox * add1.ld + c8 * 8, a);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] += a[j];
    }
    if (add2.hi) {
      float a[8];
      load8(add2.hi, add2.lo, vox * add2.ld + c8 * 8, a);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] += a[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] *= ks[j];
    store8(dx.hi, dx.lo, vox * dx.ld + c8 * 8, o);
  };
  long long s = (long long)blockIdx.x * vper + vslot;
  for (; s + stride < S; s += 2 * stride) {
    float g0[8], v0[8], g1[8], v1[8];
    load8(dz.hi, dz.lo, (base + s) * dz.ld + c8 * 8, g0);
    load8(x.hi, x.lo, (base + s) * x.ld + c8 * 8, v0);
    load8(dz.hi, dz.lo, (base + s + stride) * dz.ld + c8 * 8, g1);
    load8(x.hi, x.lo, (base + s + stride) * x.ld + c8 * 8, v1);
    one(base + s, g0, v0);
    one(base + s + stride, g1, v1);
  }
  if (s < S) {
    float g0[8], v0[8];
    load8(dz.hi, dz.lo, (base + s) * dz.ld + c8 * 8, g0);
    load8(x.hi, x.lo, (base + s) * x.ld + c8 * 8, v0);
    one(base + s, g0, v0);
  }
}

// backward statistics -> (E, F), dgamma, dbeta -> dx = A dz + E x + F (+adds)(*scale) in one launch
int launch_gn_bwd(const Act& dz, const Act& x, const float* coef, const double* bstats, const float* gamma, int C, int G,
                  long long S, float* dgamma, float* dbeta, const Act* add1, const Act* add2, const Act& dx,
                  const float* scale, cudaStream_t st) {
  B200_REQUIRE(x.C % 8 == 0 && dz.C == x.C && dx.C == x.C, E_INVALID, "gn_bwd: channel mismatch");
  B200_REQUIRE(G > 0 && C % G == 0 && C <= x.C, E_INVALID, "gn_bwd: C=%d G=%d", C, G);
  B200_REQUIRE(x.C <= 1024, E_UNSUPPORTED, "gn_bwd: C <= 1024 supported (got %d)", x.C);
  GnBwdFin f;
  f.bstats = bstats; f.gamma = gamma; f.C = C; f.G = G; f.N = x.N; f.S = (double)S; f.dgamma = dgamma; f.dbeta = dbeta;
  const Act none = make_act(nullptr, nullptr, 0, 0, 0, 0, 0, 0);
  dim3 grid, block;
  gn_launch_dims(x, grid, block);
  launch_pdl(k_gn_bwd, grid, block, 0, st, dz, x, reinterpret_cast<const float4*>(coef), add1 ? *add1 : none,
             add2 ? *add2 : none, dx, scale, f);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// ------------------------------------------------------------------------------------------------ activation backward (+ statistics)
// Post-activation blocks (conv -> norm -> act: MONAI UnetBasicBlock, the model examples/brats2020/brats2020_config.json
// trains): the gradient arriving at a block output is that of the ACTIVATED tensor a = act(A c + B), c = the
// convolution output.   dz = (g1 [+ g2]) * act'(A c + B);   bstats[n][ch] += (sum dz, sum dz * xhat),  xhat = (c - mu) rstd
// which is exactly what the GroupNorm backward (k_gn_bwd) consumes.  Same thread <-> channel-chunk mapping as k_gn_apply.
__global__ void __launch_bounds__(256) k_act_bwd(Act g1, Act g2, Act c, const float4* __restrict__ coef, float slope, Act dz,
                                                 double* __restrict__ bstats, int bstats_ld) {
  extern __shared__ double smb[];   // [C][2]
  for (int i = threadIdx.x; i < c.C * 2; i += blockDim.x) smb[i] = 0.0;
  __syncthreads();
  const int c8n = c.C / 8;
  const int n = blockIdx.y;
  const long long S = (long long)c.D * c.H * c.W;
  const int c8 = threadIdx.x % c8n;
  const int vslot = threadIdx.x / c8n, vper = blockDim.x / c8n;
  float ka[8], kb[8], km[8], kr[8], s1[8], s2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 k = __ldg(coef + (long long)n * c.C + c8 * 8 + j);
    ka[j] = k.x; kb[j] = k.y; km[j] = k.z; kr[j] = k.w;
    s1[j] = s2[j] = 0.f;
  }
  const long long base = (long long)n * S;
  for (long long s = (long long)blockIdx.x * vper + vslot; s < S; s += (long long)gridDim.x * vper) {
    float g[8], x[8];
    load8(g1.hi, g1.lo, (base + s) * g1.ld + c8 * 8, g);
    load8(c.hi, c.lo, (base + s) * c.ld + c8 * 8, x);
    if (g2.hi) {
      float h[8];
      load8(g2.hi, g2.lo, (base + s) * g2.ld + c8 * 8, h);
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] += h[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float z = fmaf(ka[j], x[j], kb[j]);
      const float d = z > 0.f ? g[j] : g[j] * slope;
      g[j] = d;
      s1[j] += d;
      s2[j] = fmaf(d, (x[j] - km[j]) * kr[j], s2[j]);
    }
    store8(dz.hi, dz.lo, (base + s) * dz.ld + c8 * 8, g);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    atomicAdd(&smb[(c8 * 8 + j) * 2 + 0], (double)s1[j]);
    atomicAdd(&smb[(c8 * 8 + j) * 2 + 1], (double)s2[j]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < c.C * 2; i += blockDim.x) atomicAdd(&bstats[(long long)n * bstats_ld * 2 + i], smb[i]);
}

int launch_act_bwd(const Act& g1, const Act* g2, const Act& c, const float* coef, float slope, const Act& dz, double* bstats,
                   int bstats_ld, cudaStream_t st) {
  B200_REQUIRE(c.C % 8 == 0 && g1.C == c.C && dz.C == c.C && (!g2 || g2->C == c.C), E_INVALID, "act_bwd: channel mismatch");
  B200_REQUIRE(coef && bstats, E_INVALID, "act_bwd: null argument");
  const int c8n = c.C / 8;
  const int threads = ew_threads_for(c8n);
  B200_REQUIRE(threads <= 256, E_UNSUPPORTED, "act_bwd: C=%d unsupported", c.C);
  const long long S = (long long)c.D * c.H * c.W;
  const int vper = threads / c8n;
  long long want = (S + vper - 1) / vper;
  const long long cap = (132LL * 4 + c.N - 1) / c.N;
  const int blocks = (int)(want < cap ? (want > 0 ? want : 1) : cap);
  Act none = make_act(nullptr, nullptr, 0, 0, 0, 0, 0, 0);
  k_act_bwd<<<dim3(blocks, c.N), threads, c.C * 2 * sizeof(double), st>>>(g1, g2 ? *g2 : none, c, reinterpret_cast<const float4*>(coef),
                                                                          slope, dz, bstats, bstats_ld);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// dbias[o] = sum over n, voxels of dlogits[n][o][s]   (bias of the 1x1x1 output block, MONAI UnetOutBlock)
// Two launches, no floating-point atomics: per-block fp64 partial sums into `part` [NO][blocks], then one thread per output adds
// them in a fixed order (a float atomicAdd per block made this the one run-to-run varying gradient of a deterministic plan).
__global__ void k_head_dbias(const float* __restrict__ dlogits, int N, int NO, long long S, double* __restrict__ part) {
  __shared__ double sh[32];
  const int o = blockIdx.y;
  double acc = 0;
  for (int n = 0; n < N; ++n) {
    const float* p = dlogits + ((long long)n * NO + o) * S;
    float a = 0.f;
    for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (long long)gridDim.x * blockDim.x) a += p[s];
    acc += (double)a;
  }
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += sh[i];
    part[(size_t)o * gridDim.x + blockIdx.x] = t;
  }
}

__global__ void k_head_dbias_sum(const double* __restrict__ part, int blocks, int NO, float* __restrict__ dbias) {
  const int o = threadIdx.x;
  if (o >= NO) return;
  double t = 0;
  for (int i = 0; i < blocks; ++i) t += part[(size_t)o * blocks + i];
  dbias[o] = (float)t;
}

// scratch: >= 128 * NO doubles (the head's weight-gradient slot arena, head_bwd_scratch_bytes(), is free again by now)
int launch_head_dbias(const float* dlogits, int N, int NO, long long S, float* dbias, cudaStream_t st, float* scratch) {
  B200_REQUIRE(scratch != nullptr && NO >= 1 && NO <= 32, E_INVALID, "head_dbias: needs scratch, 1 <= n_outputs <= 32");
  long long want = (S + 255) / 256;
  const int blocks = (int)(want < 128 ? (want > 0 ? want : 1) : 128);
  double* part = reinterpret_cast<double*>(scratch);
  k_head_dbias<<<dim3(blocks, NO), 256, 0, st>>>(dlogits, N, NO, S, part);
  B200_CHECK_CUDA(cudaGetLastError());
  k_head_dbias_sum<<<1, 32, 0, st>>>(part, blocks, NO, dbias);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// ------------------------------------------------------------------------------------------------ trilinear x2 (align_corners=False)
// out[2k] = .25 x[clamp(k-1)] + .75 x[k] ; out[2k+1] = .75 x[k] + .25 x[clamp(k+1)]   per axis (separable).
// Output is written into a channel slice view (concat fusion) and its per-channel statistics are accumulated.
__device__ __forceinline__ void up_taps(int o, int n, int& i0, int& i1, float& w0, float& w1) {
  const int k = o >> 1;
  if (o & 1) { i0 = k; i1 = k + 1 < n ? k + 1 : n - 1; w0 = 0.75f; w1 = 0.25f; }
  else       { i0 = k - 1 >= 0 ? k - 1 : 0; i1 = k; w0 = 0.25f; w1 = 0.75f; }
}

// Each thread produces a 2x2x2 block of outputs (o = 2k+1, 2k+2 per axis, k in [-1, n-1]) from the 2x2x2 block of
// inputs (clamp(k), clamp(k+1)): 8 loads for 8 outputs instead of 8 loads per output.  grid (blocks, N); the 8-channel
// chunk is constant per thread, so the per-channel statistics accumulate in registers.
// ADD: y = upsample(x) + add (SegResNet's additive skip), the statistics taken of the sum; one full-resolution write and
// re-read fewer than an up-sampling followed by an add.
template <bool ADD>
__global__ void __launch_bounds__(256) k_upsample2x_fwd(Act x, Act y, double* __restrict__ stats, int stats_ld, Act add) {
  const int c8n = x.C / 8;
  extern __shared__ double smu[];  // [C][2], fp64: atomic order must not reach the fp32 coefficients
  if (stats) {
    for (int i = threadIdx.x; i < x.C * 2; i += blockDim.x) smu[i] = 0.0;
    __syncthreads();
  }
  const int n = blockIdx.y;
  const int c8 = threadIdx.x % c8n;
  const int vslot = threadIdx.x / c8n;
  const int vper = blockDim.x / c8n;
  const int bw = x.W + 1, bh = x.H + 1, bd = x.D + 1;
  const int nblk = bw * bh * bd;
  float a[8], b[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) a[j] = b[j] = 0.f;
  for (int t = blockIdx.x * vper + vslot; t < nblk; t += gridDim.x * vper) {
    const int kw = t % bw - 1, kh = (t / bw) % bh - 1, kd = t / (bw * bh) - 1;
    const int w0 = kw < 0 ? 0 : kw, w1 = kw + 1 < x.W ? kw + 1 : x.W - 1;
    const int h0 = kh < 0 ? 0 : kh, h1 = kh + 1 < x.H ? kh + 1 : x.H - 1;
    const int d0 = kd < 0 ? 0 : kd, d1 = kd + 1 < x.D ? kd + 1 : x.D - 1;
    float v[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int d = (i & 4) ? d1 : d0, h = (i & 2) ? h1 : h0, w = (i & 1) ? w1 : w0;
      load8(x.hi, x.lo, ((((long long)n * x.D + d) * x.H + h) * x.W + w) * x.ld + c8 * 8, v[i]);
    }
#pragma unroll
    for (int o = 0; o < 8; ++o) {
      const int od = 2 * kd + 1 + ((o >> 2) & 1), oh = 2 * kh + 1 + ((o >> 1) & 1), ow = 2 * kw + 1 + (o & 1);
      if (od < 0 || oh < 0 || ow < 0 || od >= y.D || oh >= y.H || ow >= y.W) continue;
      // output 2k+1 = .75 x[k] + .25 x[k+1] ; output 2k+2 = .25 x[k] + .75 x[k+1]
      const float wd1 = (o & 4) ? 0.75f : 0.25f, wh1 = (o & 2) ? 0.75f : 0.25f, ww1 = (o & 1) ? 0.75f : 0.25f;
      float r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float wt = ((i & 4) ? wd1 : 1.f - wd1) * ((i & 2) ? wh1 : 1.f - wh1) * ((i & 1) ? ww1 : 1.f - ww1);
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = fmaf(wt, v[i][j], r[j]);
      }
      if (ADD) {
        float s[8];
        load8(add.hi, add.lo, ((((long long)n * add.D + od) * add.H + oh) * add.W + ow) * add.ld + c8 * 8, s);
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] += s[j];
      }
      store8(y.hi, y.lo, ((((long long)n * y.D + od) * y.H + oh) * y.W + ow) * y.ld + c8 * 8, r);
#pragma unroll
      for (int j = 0; j < 8; ++j) { a[j] += r[j]; b[j] = fmaf(r[j], r[j], b[j]); }
    }
  }
  if (stats) {
    const bool pow2 = (c8n & (c8n - 1)) == 0 && c8n <= 32;   // then lanes l, l' share the chunk iff l % c8n == l' % c8n
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float pa = a[j], pb = b[j];
      if (pow2) {
        for (int off = 16; off >= c8n; off >>= 1) {
          pa += __shfl_xor_sync(0xffffffffu, pa, off);
          pb += __shfl_xor_sync(0xffffffffu, pb, off);
        }
        if ((threadIdx.x & 31) < c8n) {
          atomicAdd(&smu[(c8 * 8 + j) * 2 + 0], (double)pa);
          atomicAdd(&smu[(c8 * 8 + j) * 2 + 1], (double)pb);
        }
      } else {
        atomicAdd(&smu[(c8 * 8 + j) * 2 + 0], (double)pa);
        atomicAdd(&smu[(c8 * 8 + j) * 2 + 1], (double)pb);
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < x.C * 2; i += blockDim.x) atomicAdd(&stats[(long long)n * stats_ld * 2 + i], smu[i]);
  }
}

int launch_upsample2x_fwd(const Act& x, const Act& y, double* stats, int stats_ld, cudaStream_t st, const Act* add) {
  B200_REQUIRE(x.C % 8 == 0 && y.C == x.C, E_INVALID, "upsample: channel mismatch");
  B200_REQUIRE(y.D == 2 * x.D && y.H == 2 * x.H && y.W == 2 * x.W, E_UNSUPPORTED,
               "upsample: output must be exactly 2x (got %dx%dx%d -> %dx%dx%d)", x.D, x.H, x.W, y.D, y.H, y.W);
  if (add)
    B200_REQUIRE(add->N == y.N && add->D == y.D && add->H == y.H && add->W == y.W && add->C == y.C && add->ld % 8 == 0, E_INVALID,
                 "upsample: the addend must have the output's shape (%dx%dx%dx%dx%d, got %dx%dx%dx%dx%d)", y.N, y.D, y.H, y.W, y.C,
                 add->N, add->D, add->H, add->W, add->C);
  const int c8n = x.C / 8;
  const int threads = ew_threads_for(c8n);
  B200_REQUIRE(threads <= 256, E_UNSUPPORTED, "upsample: C=%d unsupported (at most 2048 channels)", x.C);
  const int vper = threads / c8n;
  const long long nblk = (long long)(x.D + 1) * (x.H + 1) * (x.W + 1);
  B200_REQUIRE(nblk < (1LL << 31), E_UNSUPPORTED, "upsample: volume too large");
  long long want = (nblk + vper - 1) / vper;
  // at most 4 blocks per SM for EACH sample, whatever the batch (the grid of a batch of two is unchanged): the blocks' fp32
  // partial sums of the statistics then cover the same voxels at every batch size, so a sample's statistics, and its outputs,
  // do not depend on what else is in the batch
  const long long cap = 132LL * 4;
  const int blocks = (int)(want < cap ? (want > 0 ? want : 1) : cap);
  if (add) k_upsample2x_fwd<true><<<dim3(blocks, x.N), threads, x.C * 2 * sizeof(double), st>>>(x, y, stats, stats_ld, *add);
  else k_upsample2x_fwd<false><<<dim3(blocks, x.N), threads, x.C * 2 * sizeof(double), st>>>(x, y, stats, stats_ld, Act());
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// adjoint: dx[k] = .75 dy[2k] + .75 dy[2k+1] + .25 dy[2k-1] (k>=1) + .25 dy[2k+2] (k<=n-2) + clamp terms
__device__ __forceinline__ int up_adj(int k, int n, int (&idx)[4], float (&w)[4]) {
  int cnt = 0;
  idx[cnt] = 2 * k; w[cnt] = 0.75f; ++cnt;
  idx[cnt] = 2 * k + 1; w[cnt] = 0.75f; ++cnt;
  if (k >= 1) { idx[cnt] = 2 * k - 1; w[cnt] = 0.25f; ++cnt; } else { w[0] += 0.25f; }            // out[0] clamps to x[0]
  if (k + 1 <= n - 1) { idx[cnt] = 2 * k + 2; w[cnt] = 0.25f; ++cnt; } else { w[1] += 0.25f; }  // out[2n-1] clamps to x[n-1]
  return cnt;
}

__global__ void k_upsample2x_bwd(Act dy, Act dx) {
  const int c8n = dx.C / 8;
  const long long total = dx.voxels() * c8n;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(t % c8n);
    long long v = t / c8n;
    const int w = (int)(v % dx.W); v /= dx.W;
    const int h = (int)(v % dx.H); v /= dx.H;
    const int d = (int)(v % dx.D);
    const int n = (int)(v / dx.D);
    int id[4], ih[4], iw[4]; float wd[4], wh[4], ww[4];
    const int nd = up_adj(d, dx.D, id, wd), nh = up_adj(h, dx.H, ih, wh), nw = up_adj(w, dx.W, iw, ww);
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = 0.f;
    for (int a = 0; a < nd; ++a)
      for (int b = 0; b < nh; ++b)
        for (int c = 0; c < nw; ++c) {
          const float wt = wd[a] * wh[b] * ww[c];
          float g[8];
          load8(dy.hi, dy.lo, ((((long long)n * dy.D + id[a]) * dy.H + ih[b]) * dy.W + iw[c]) * dy.ld + c8 * 8, g);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = fmaf(wt, g[j], o[j]);
        }
    store8(dx.hi, dx.lo, ((((long long)n * dx.D + d) * dx.H + h) * dx.W + w) * dx.ld + c8 * 8, o);
  }
}

// Register-blocked form (single-pass bf16, even extents): a thread owns a 2 x 2 x 2 block of dx voxels (8 channels) and walks the
// 6 x 6 x 6 neighbourhood of dy once -- 216 16-byte loads per 8 outputs instead of 8 x 64: the gather form above is bound by
// L1/L2 load bandwidth (8x read amplification), not by HBM.  Per axis, block m (outputs 2m, 2m+1) meets dy indices 4m-1+i,
// i = 0..5: output 2m with weights (.25 .75 .75 .25) on i = 0..3, output 2m+1 with the same on i = 2..5; a neighbour outside
// the volume hands its weight to the clamped one (i = 0 when m = 0, i = 5 at the far end).
__device__ __forceinline__ float blk_w0(int i, bool first) {
  return i == 0 ? (first ? 0.f : 0.25f) : i == 1 ? (first ? 1.0f : 0.75f) : i == 2 ? 0.75f : i == 3 ? 0.25f : 0.f;
}
__device__ __forceinline__ float blk_w1(int i, bool last) {
  return i == 2 ? 0.25f : i == 3 ? 0.75f : i == 4 ? (last ? 1.0f : 0.75f) : i == 5 ? (last ? 0.f : 0.25f) : 0.f;
}

__global__ void __launch_bounds__(128) k_upsample2x_bwd_blk(Act dy, Act dx) {
  const int c8n = dx.C / 8;
  const int bw = dx.W >> 1, bh = dx.H >> 1, bd = dx.D >> 1;
  const long long total = (long long)dx.N * bd * bh * bw * c8n;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(t % c8n);
    long long v = t / c8n;
    const int mw = (int)(v % bw); v /= bw;
    const int mh = (int)(v % bh); v /= bh;
    const int md = (int)(v % bd);
    const int n = (int)(v / bd);
    const bool fw = mw == 0, lw = mw == bw - 1, fh = mh == 0, lh = mh == bh - 1, fd = md == 0, ld_ = md == bd - 1;
    float wx0[4], wx1[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { wx0[i] = blk_w0(i, fw); wx1[i] = blk_w1(i + 2, lw); }
    float o[2][2][2][8];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int c = 0; c < 2; ++c)
#pragma unroll
          for (int j = 0; j < 8; ++j) o[a][b][c][j] = 0.f;
    const bf16* base = dy.hi + (long long)n * dy.D * dy.H * dy.W * dy.ld + c8 * 8;
#pragma unroll 1
    for (int iz = 0; iz < 6; ++iz) {
      const float wz0 = blk_w0(iz, fd), wz1 = blk_w1(iz, ld_);
      if (wz0 == 0.f && wz1 == 0.f) continue;           // the plane lies outside the volume
      const int gz = 4 * md - 1 + iz;
#pragma unroll 1
      for (int iy = 0; iy < 6; ++iy) {
        const float wy0 = blk_w0(iy, fh), wy1 = blk_w1(iy, lh);
        if (wy0 == 0.f && wy1 == 0.f) continue;
        const int gy = 4 * mh - 1 + iy;
        const bf16* row = base + (((long long)gz * dy.H + gy) * dy.W + 4 * mw - 1) * dy.ld;
        float r0[8], r1[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { r0[j] = 0.f; r1[j] = 0.f; }
#pragma unroll
        for (int ix = 0; ix < 6; ++ix) {
          if ((ix == 0 && fw) || (ix == 5 && lw)) continue;
          const uint4 a = *reinterpret_cast<const uint4*>(row + (long long)ix * dy.ld);
          float g[8];
          g[0] = bf16_lo_to_f(a.x); g[1] = bf16_hi_to_f(a.x); g[2] = bf16_lo_to_f(a.y); g[3] = bf16_hi_to_f(a.y);
          g[4] = bf16_lo_to_f(a.z); g[5] = bf16_hi_to_f(a.z); g[6] = bf16_lo_to_f(a.w); g[7] = bf16_hi_to_f(a.w);
          if (ix < 4) {
#pragma unroll
            for (int j = 0; j < 8; ++j) r0[j] = fmaf(wx0[ix], g[j], r0[j]);
          }
          if (ix >= 2) {
#pragma unroll
            for (int j = 0; j < 8; ++j) r1[j] = fmaf(wx1[ix - 2], g[j], r1[j]);
          }
        }
        const float w00 = wz0 * wy0, w01 = wz0 * wy1, w10 = wz1 * wy0, w11 = wz1 * wy1;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          o[0][0][0][j] = fmaf(w00, r0[j], o[0][0][0][j]); o[0][0][1][j] = fmaf(w00, r1[j], o[0][0][1][j]);
          o[0][1][0][j] = fmaf(w01, r0[j], o[0][1][0][j]); o[0][1][1][j] = fmaf(w01, r1[j], o[0][1][1][j]);
          o[1][0][0][j] = fmaf(w10, r0[j], o[1][0][0][j]); o[1][0][1][j] = fmaf(w10, r1[j], o[1][0][1][j]);
          o[1][1][0][j] = fmaf(w11, r0[j], o[1][1][0][j]); o[1][1][1][j] = fmaf(w11, r1[j], o[1][1][1][j]);
        }
      }
    }
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int c = 0; c < 2; ++c)
          store8(dx.hi, nullptr, ((((long long)n * dx.D + 2 * md + a) * dx.H + 2 * mh + b) * dx.W + 2 * mw + c) * dx.ld + c8 * 8, o[a][b][c]);
  }
}

int launch_upsample2x_bwd(const Act& dy, const Act& dx, cudaStream_t st) {
  B200_REQUIRE(dx.C % 8 == 0 && dy.C == dx.C, E_INVALID, "upsample_bwd: channel mismatch");
  B200_REQUIRE(dy.D == 2 * dx.D && dy.H == 2 * dx.H && dy.W == 2 * dx.W, E_UNSUPPORTED, "upsample_bwd: not 2x");
  if (!dy.lo && !dx.lo && dx.D % 2 == 0 && dx.H % 2 == 0 && dx.W % 2 == 0 && dx.D >= 2 && dx.H >= 2 && dx.W >= 2) {
    const long long blocks = (long long)dx.N * (dx.D / 2) * (dx.H / 2) * (dx.W / 2) * (dx.C / 8);
    k_upsample2x_bwd_blk<<<ew_blocks(blocks, 128), 128, 0, st>>>(dy, dx);
    B200_CHECK_CUDA(cudaGetLastError());
    return OK;
  }
  long long total = dx.voxels() * (dx.C / 8);
  k_upsample2x_bwd<<<ew_blocks(total, 256), 256, 0, st>>>(dy, dx);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// ------------------------------------------------------------------------------------------------ head: 1x1x1 conv C -> n_out
// logits NCDHW fp32 (the reference-facing layout).  One thread per voxel; weights in shared memory.
__global__ void k_head_fwd(Act x, const float* __restrict__ w, const float* __restrict__ bias, int n_out, int act_mode,
                           float* __restrict__ logits) {
  extern __shared__ float sw[];  // [n_out][C]
  for (int i = threadIdx.x; i < n_out * x.C; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const long long S = (long long)x.D * x.H * x.W;
  const long long total = x.N * S;
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < total; v += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(v / S);
    const long long s = v % S;
    float acc[8];
#pragma unroll
    for (int o = 0; o < 8; ++o) acc[o] = (bias && o < n_out) ? __ldg(bias + o) : 0.f;
    for (int c0 = 0; c0 < x.C; c0 += 8) {
      float u[8];
      load8(x.hi, x.lo, v * x.ld + c0, u);
#pragma unroll
      for (int o = 0; o < 8; ++o)
        if (o < n_out) {
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[o] = fmaf(sw[o * x.C + c0 + j], u[j], acc[o]);
        }
    }
    if (act_mode == 2) {  // softmax over channels
      float m = -INFINITY;
      for (int o = 0; o < n_out; ++o) m = fmaxf(m, acc[o]);
      float z = 0.f;
      for (int o = 0; o < n_out; ++o) { acc[o] = __expf(acc[o] - m); z += acc[o]; }
      for (int o = 0; o < n_out; ++o) acc[o] /= z;
    }
    for (int o = 0; o < n_out; ++o) {
      float r = acc[o];
      if (act_mode == 1) r = 1.f / (1.f + __expf(-r));
      logits[((long long)n * n_out + o) * S + s] = r;
    }
  }
}

int launch_head_fwd(const Act& x, const float* w, int n_out, int act_mode, float* logits, cudaStream_t st, const float* bias) {
  if (n_out > 8) return launch_head_mma_fwd(x, w, n_out, act_mode, logits, st, bias);
  B200_REQUIRE(n_out >= 1, E_UNSUPPORTED, "head: n_outputs=%d unsupported (1..%d)", n_out, B200_HEAD_MAX_OUTPUTS);
  B200_REQUIRE(x.C % 8 == 0, E_INVALID, "head: C=%d", x.C);
  k_head_fwd<<<ew_blocks(x.voxels(), 256), 256, n_out * x.C * sizeof(float), st>>>(x, w, bias, n_out, act_mode, logits);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// dx[v][c] = sum_o dlogits[n][o][s] * w[o][c] ;  dw[o][c] += sum_v dlogits[o] * x[v][c]
// thread <-> (voxel, 8-channel chunk): the chunk is fixed per thread across the grid-stride loop, so the dw partials
// (n_out x 8) stay in registers and are reduced once at the end (shuffle over lanes that share the chunk -> smem -> global).
template <int NO>
__global__ void k_head_bwd(Act x, const float* __restrict__ w, const float* __restrict__ dlogits, Act dx,
                           float* __restrict__ part) {
  extern __shared__ float sm[];  // sw [NO][C] | sdw [NO][C]
  float* sw = sm;
  float* sdw = sm + NO * x.C;
  for (int i = threadIdx.x; i < NO * x.C; i += blockDim.x) { sw[i] = w[i]; sdw[i] = 0.f; }
  __syncthreads();
  const int c8n = x.C / 8;
  const long long S = (long long)x.D * x.H * x.W;
  const long long total = (long long)x.N * S * c8n;
  const int c8 = threadIdx.x % c8n;   // blockDim.x % c8n == 0 and the grid stride is a multiple of blockDim.x
  float pdw[NO][8];
#pragma unroll
  for (int o = 0; o < NO; ++o)
#pragma unroll
    for (int j = 0; j < 8; ++j) pdw[o][j] = 0.f;
  float wr[NO][8];
#pragma unroll
  for (int o = 0; o < NO; ++o)
#pragma unroll
    for (int j = 0; j < 8; ++j) wr[o][j] = sw[o * x.C + c8 * 8 + j];
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const long long v = t / c8n;
    const int n = (int)(v / S);
    const long long s = v % S;
    float g[NO];
#pragma unroll
    for (int o = 0; o < NO; ++o) g[o] = __ldg(dlogits + ((long long)n * NO + o) * S + s);
    float u[8], d[8];
    load8(x.hi, x.lo, v * x.ld + c8 * 8, u);
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] = 0.f;
#pragma unroll
    for (int o = 0; o < NO; ++o)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        d[j] = fmaf(g[o], wr[o][j], d[j]);
        pdw[o][j] = fmaf(g[o], u[j], pdw[o][j]);
      }
    store8(dx.hi, dx.lo, v * dx.ld + c8 * 8, d);
  }
  // Block reduction in a FIXED order (no floating-point atomics): per-thread partials -> shared memory -> thread i sums the
  // threads that own channel i's chunk (t = c8, c8 + c8n, ...) -> this block's slot of `part`; k_sum_slots then adds the
  // block slots in order.  The weight gradient of the head is bit-reproducible run to run.
  float* s_tmp = sdw + NO * x.C;   // [blockDim.x][8]
#pragma unroll
  for (int o = 0; o < NO; ++o) {
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) s_tmp[threadIdx.x * 8 + j] = pdw[o][j];
    __syncthreads();
    for (int i = threadIdx.x; i < x.C; i += blockDim.x) {
      const int ch = i >> 3, j = i & 7;
      float acc = 0.f;
      for (int t = ch; t < (int)blockDim.x; t += c8n) acc += s_tmp[t * 8 + j];
      part[(long long)blockIdx.x * NO * x.C + o * x.C + i] = acc;
    }
  }
}

// out[i] = sum over slots of part[s][i], one block per i, in a FIXED order: thread t adds the slots t, t + 128, ... and a
// shared-memory tree combines the 128 partial sums (a single thread walking all ~1200 slots took 0.07 ms of pure load latency)
__global__ void __launch_bounds__(128) k_sum_slots(const float* __restrict__ part, int slots, int n, float* __restrict__ out) {
  __shared__ float s_acc[128];
  const int i = blockIdx.x;
  float acc = 0.f;
  for (int s = threadIdx.x; s < slots; s += 128) acc += part[(long long)s * n + i];
  s_acc[threadIdx.x] = acc;
  __syncthreads();
  for (int h = 64; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) s_acc[threadIdx.x] += s_acc[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[i] = s_acc[0];
}

size_t head_bwd_scratch_bytes(int n_out, int C) {
  return n_out > 8 ? head_mma_bwd_scratch_bytes(n_out, C) : (size_t)1184 * n_out * C * sizeof(float);
}

int launch_head_bwd(const Act& x, const float* w, int n_out, const float* dlogits, const Act& dx, float* dw,
                    cudaStream_t st, float* scratch, float* dbias) {
  B200_REQUIRE(scratch != nullptr, E_INVALID, "head_bwd: needs head_bwd_scratch_bytes() of scratch");
  if (n_out > 8) {   // one pass writes dx and the per-CTA partials of dw (and dbias); fixed-order slot sums follow
    int slots = 0;
    B200_TRY(launch_head_mma_bwd(x, w, n_out, dlogits, dx, dbias != nullptr, scratch, &slots, st));
    k_sum_slots<<<n_out * x.C, 128, 0, st>>>(scratch, slots, n_out * x.C, dw);
    B200_CHECK_CUDA(cudaGetLastError());
    if (dbias) {
      k_sum_slots<<<n_out, 128, 0, st>>>(scratch + (size_t)slots * n_out * x.C, slots, n_out, dbias);
      B200_CHECK_CUDA(cudaGetLastError());
    }
    return OK;
  }
  B200_REQUIRE(n_out >= 1, E_UNSUPPORTED, "head_bwd: n_outputs=%d unsupported (1..%d)", n_out, B200_HEAD_MAX_OUTPUTS);
  B200_REQUIRE(dbias == nullptr, E_INVALID, "head_bwd: the bias gradient of 1..8 outputs comes from launch_head_dbias");
  B200_REQUIRE(x.C % 8 == 0 && dx.C == x.C, E_INVALID, "head_bwd: channel mismatch");
  const int c8n = x.C / 8;
  int threads = 256;
  while (threads % c8n) threads += 32;
  B200_REQUIRE(threads <= 1024, E_UNSUPPORTED, "head_bwd: C=%d unsupported", x.C);
  long long total = x.voxels() * c8n;
  int blocks = ew_blocks(total, threads);
  if (blocks > 1184) blocks = 1184;
  const size_t smem = (2 * n_out * x.C + (size_t)threads * 8) * sizeof(float);
#define B200_HEAD_CASE(no) \
  case no: k_head_bwd<no><<<blocks, threads, smem, st>>>(x, w, dlogits, dx, scratch); break;
  switch (n_out) {
    B200_HEAD_CASE(1) B200_HEAD_CASE(2) B200_HEAD_CASE(3) B200_HEAD_CASE(4)
    B200_HEAD_CASE(5) B200_HEAD_CASE(6) B200_HEAD_CASE(7) B200_HEAD_CASE(8)
  }
#undef B200_HEAD_CASE
  B200_CHECK_CUDA(cudaGetLastError());
  k_sum_slots<<<n_out * x.C, 128, 0, st>>>(scratch, blocks, n_out * x.C, dw);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// ------------------------------------------------------------------------------------------------ bias gradient
// dbias[c] = sum over the visible voxels (d < vD, h < vH, w < vW) of dy[v][c]   (ConvTranspose3d bias; the padded
// boundary of its output is a constant and carries no gradient)
// No floating-point atomics, so that a deterministic plan repeats this gradient bit for bit: each block sums its threads'
// partials in a fixed order into its slot of `part` [blocks][C] (as k_head_bwd does), then k_sum_slots adds the slots in order.
constexpr int kBiasGradSlots = 592;
__global__ void k_bias_grad(Act dy, float* __restrict__ part) {
  const int c8n = dy.C / 8;
  const int c8 = threadIdx.x % c8n;
  const int vslot = threadIdx.x / c8n, vper = blockDim.x / c8n;
  const int vD = dy.vD > 0 ? dy.vD : dy.D, vH = dy.vH > 0 ? dy.vH : dy.H, vW = dy.vW > 0 ? dy.vW : dy.W;
  const long long total = dy.voxels();
  float a[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) a[j] = 0.f;
  for (long long v = (long long)blockIdx.x * vper + vslot; v < total; v += (long long)gridDim.x * vper) {
    const int w = (int)(v % dy.W), h = (int)((v / dy.W) % dy.H), d = (int)((v / ((long long)dy.W * dy.H)) % dy.D);
    if (w >= vW || h >= vH || d >= vD) continue;
    float g[8];
    load8(dy.hi, dy.lo, v * dy.ld + c8 * 8, g);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += g[j];
  }
  extern __shared__ float s_tmp[];   // [blockDim.x][8]
#pragma unroll
  for (int j = 0; j < 8; ++j) s_tmp[threadIdx.x * 8 + j] = a[j];
  __syncthreads();
  for (int i = threadIdx.x; i < dy.C; i += blockDim.x) {
    float acc = 0.f;
    for (int t = i >> 3; t < (int)blockDim.x; t += c8n) acc += s_tmp[t * 8 + (i & 7)];
    part[(long long)blockIdx.x * dy.C + i] = acc;
  }
}

size_t bias_grad_scratch_bytes(int C) { return (size_t)kBiasGradSlots * C * sizeof(float); }

int launch_bias_grad(const Act& dy, float* dbias, float* scratch, cudaStream_t st) {
  B200_REQUIRE(dy.C % 8 == 0, E_INVALID, "bias_grad: C=%d", dy.C);
  B200_REQUIRE(scratch != nullptr, E_INVALID, "bias_grad: needs bias_grad_scratch_bytes() of scratch");
  const int threads = ew_threads_for(dy.C / 8);
  B200_REQUIRE(threads <= 1024, E_UNSUPPORTED, "bias_grad: C=%d unsupported", dy.C);
  long long want = (dy.voxels() + threads / (dy.C / 8) - 1) / (threads / (dy.C / 8));
  int blocks = (int)(want < kBiasGradSlots ? (want > 0 ? want : 1) : kBiasGradSlots);
  k_bias_grad<<<blocks, threads, (size_t)threads * 8 * sizeof(float), st>>>(dy, scratch);
  B200_CHECK_CUDA(cudaGetLastError());
  k_sum_slots<<<dy.C, 128, 0, st>>>(scratch, blocks, dy.C, dbias);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// ------------------------------------------------------------------------------------------------ zero insertion (x2 dilation)
// z[2d+od][2h+oh][2w+ow] = x[d][h][w], zeros elsewhere; z dims given by the view (>= 2*x dims - 1 + offset).
__global__ void k_zero_insert(Act x, Act z, int od, int oh, int ow) {
  const int c8n = z.C / 8;
  const long long total = z.voxels() * c8n;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(t % c8n);
    long long v = t / c8n;
    const int w = (int)(v % z.W); v /= z.W;
    const int h = (int)(v % z.H); v /= z.H;
    const int d = (int)(v % z.D);
    const int n = (int)(v / z.D);
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = 0.f;
    const int sd = d - od, sh = h - oh, sw = w - ow;
    if (sd >= 0 && sh >= 0 && sw >= 0 && !(sd & 1) && !(sh & 1) && !(sw & 1) && (sd >> 1) < x.D && (sh >> 1) < x.H &&
        (sw >> 1) < x.W)
      load8(x.hi, x.lo, ((((long long)n * x.D + (sd >> 1)) * x.H + (sh >> 1)) * x.W + (sw >> 1)) * x.ld + c8 * 8, o);
    store8(z.hi, z.lo, (t / c8n) * z.ld + c8 * 8, o);
  }
}

int launch_zero_insert(const Act& x, const Act& z, int od, int oh, int ow, cudaStream_t st) {
  B200_REQUIRE(x.C == z.C && x.C % 8 == 0, E_INVALID, "zero_insert: channel mismatch");
  long long total = z.voxels() * (z.C / 8);
  k_zero_insert<<<ew_blocks(total, 256), 256, 0, st>>>(x, z, od, oh, ow);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// ------------------------------------------------------------------------------------------------ layout converters (tests / boundary)
__global__ void k_ncdhw_to_act(const float* __restrict__ x, int C, Act out) {
  const long long S = (long long)out.D * out.H * out.W;
  const int c8n = out.C / 8;
  const long long total = out.N * S * c8n;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(t % c8n);
    const long long vox = t / c8n;
    const int n = (int)(vox / S);
    const long long s = vox % S;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { int c = c8 * 8 + j; v[j] = c < C ? x[((long long)n * C + c) * S + s] : 0.f; }
    store8(out.hi, out.lo, vox * out.ld + c8 * 8, v);
  }
}
__global__ void k_act_to_ncdhw(Act in, int C, float* __restrict__ y) {
  const long long S = (long long)in.D * in.H * in.W;
  const int c8n = in.C / 8;
  const long long total = in.N * S * c8n;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(t % c8n);
    const long long vox = t / c8n;
    const int n = (int)(vox / S);
    const long long s = vox % S;
    float v[8];
    load8(in.hi, in.lo, vox * in.ld + c8 * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) { int c = c8 * 8 + j; if (c < C) y[((long long)n * C + c) * S + s] = v[j]; }
  }
}

// ------------------------------------------------------------------------------------------------ network input gradient
// dx[n][c][s] = (A dz + E x + F) + r  for the C real channels of the network input, in ONE pass from NDHWC bf16 (hi [+ lo])
// to NCDHW fp32: the GroupNorm(+ReLU) backward of the first norm (dz is already masked by ReLU'; A from coef, (E, F) from the
// coef2 gn_bwd_finalize left behind), the residual branch r (the `sample` data gradient or the identity gradient) and the
// transpose.  dz.hi == nullptr switches the norm step off (dx = r).  A tile of kInputGradTile voxels is staged in shared
// memory: the loads are 16-byte NDHWC vectors, the stores run along W (NCDHW), both coalesced.
constexpr int kInputGradTile = 256;
__global__ void __launch_bounds__(256) k_input_grad(Act dz, Act x, const float4* __restrict__ coef, const float2* __restrict__ coef2,
                                                    int coef_ld, Act r, int C, float* __restrict__ dx) {
  __shared__ float tile[16][kInputGradTile + 1];
  __shared__ float s_a[16], s_e[16], s_f[16];
  const int n = blockIdx.y;
  const long long S = (long long)r.D * r.H * r.W;
  const long long s0 = (long long)blockIdx.x * kInputGradTile;
  const int c8n = (C + 7) / 8;
  if (threadIdx.x < 16) {
    const int c = threadIdx.x;
    const bool on = dz.hi && c < C;
    s_a[c] = on ? coef[(long long)n * coef_ld + c].x : 0.f;
    s_e[c] = on ? coef2[(long long)n * coef_ld + c].x : 0.f;
    s_f[c] = on ? coef2[(long long)n * coef_ld + c].y : 0.f;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < kInputGradTile * c8n; t += blockDim.x) {
    const int v = t / c8n, c8 = t % c8n;
    const long long s = s0 + v;
    if (s >= S) continue;
    const long long vox = (long long)n * S + s;
    float o[8];
    load8(r.hi, r.lo, vox * r.ld + c8 * 8, o);
    if (dz.hi) {
      float g[8], xv[8];
      load8(dz.hi, dz.lo, vox * dz.ld + c8 * 8, g);
      load8(x.hi, x.lo, vox * x.ld + c8 * 8, xv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = c8 * 8 + j;
        o[j] = fmaf(s_a[c], g[j], fmaf(s_e[c], xv[j], s_f[c])) + o[j];   // the order of k_gn_bwd: norm term, then the residual
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) tile[c8 * 8 + j][v] = o[j];
  }
  __syncthreads();
  for (int t = threadIdx.x; t < kInputGradTile * C; t += blockDim.x) {
    const int c = t / kInputGradTile, v = t % kInputGradTile;
    const long long s = s0 + v;
    if (s < S) dx[((long long)n * C + c) * S + s] = tile[c][v];
  }
}

int launch_input_grad(const Act* dz, const Act* x, const float* coef, const float* coef2, int coef_ld, const Act& r, int C, float* dx,
                      cudaStream_t st) {
  B200_REQUIRE(C >= 1 && C <= 16 && r.C >= round_up(C, 8) && r.ld % 8 == 0, E_INVALID, "input_grad: C=%d, residual view %d/%d", C, r.C, r.ld);
  B200_REQUIRE(!dz || (x && coef && coef2 && dz->C >= C && x->C >= C && coef_ld >= C), E_INVALID, "input_grad: norm operands");
  Act none = make_act(nullptr, nullptr, 0, 0, 0, 0, 0, 0);
  const long long S = (long long)r.D * r.H * r.W;
  const long long tiles = (S + kInputGradTile - 1) / kInputGradTile;
  B200_REQUIRE(tiles < (1LL << 31) && r.N <= 65535, E_UNSUPPORTED, "input_grad: extent too large");
  k_input_grad<<<dim3((unsigned)tiles, r.N), 256, 0, st>>>(dz ? *dz : none, dz ? *x : none, reinterpret_cast<const float4*>(coef),
                                                         reinterpret_cast<const float2*>(coef2), coef_ld, r, C, dx);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

int launch_ncdhw_to_act(const float* x, int C, const Act& out, cudaStream_t st) {
  long long total = out.voxels() * (out.C / 8);
  k_ncdhw_to_act<<<ew_blocks(total, 256), 256, 0, st>>>(x, C, out);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}
int launch_act_to_ncdhw(const Act& in, int C, float* y, cudaStream_t st) {
  long long total = in.voxels() * (in.C / 8);
  k_act_to_ncdhw<<<ew_blocks(total, 256), 256, 0, st>>>(in, C, y);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

}  // namespace b200
