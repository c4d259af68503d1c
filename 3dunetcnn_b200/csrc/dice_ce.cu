// Fused Dice + cross-entropy criterion (monai.losses.DiceCELoss), forward and backward, on label-map or C-channel targets.
//
//   loss = lambda_dice * Dice(act(x), t) + lambda_ce * CE(x, t)
//   Dice: the DiceLoss formula on p = act(x), act = softmax over channels, sigmoid or identity; per (n,c)
//         I = sum p*t, P = sum p (or p^2), T = sum t (or t^2), f = 1 - (2I + nr) / (P + T + dr)   [jaccard: 2(P + T - I)]
//         include_background = 0 drops channel 0 after the activation; batch pools the sums over n; mean or sum of f.
//         The loss and the backward coefficients are formed by dice.cu's finalize, which DiceLoss shares.
//   CE:   on the raw logits.  C > 1: -sum_c t_c log_softmax(x)_c (a label map is its one-hot row); C == 1: BCEWithLogits(x, t).
//         mean divides by N*S, sum sums.  lambda_ce = 0: no CE work at all, so logits of +-inf leave a sigmoid Dice finite
//         (0 * the NaN of inf - inf would not be).
// A label outside [0, C) is an all-zero target row: it adds nothing to I, T or CE and is never used as an index.
//
// Logits are NCDHW fp32, so every channel of a sample is a contiguous run of S floats.  Both passes stage a tile of kV voxels x
// all C channels in shared memory (cp.async, one HBM read of the logits) and compute the per-voxel softmax statistics from it
// when the CE term or a softmax needs them.
//   forward:  thread v of the tile: max, sum of exponentials, CE term; then thread (c, slice) accumulates channel c's (I, P, T)
//             over a slice of the tile's voxels in registers across the block's tiles.  Each block writes its partial sums to its
//             own slot; k_dice_ce_reduce adds the slots in a fixed order in fp64 and launch_dice_finalize forms the loss and the
//             backward coefficients.  No floating-point atomics: loss and dlogits are bit-identical run to run.
//   backward: thread v of the tile: g_c = a_nc t_c + b_nc dP/dp_c from the coefficients, the activation Jacobian
//             (softmax: p_c (g_c - sum_k p_k g_k)) and the CE gradient cg (q_c sum_k t_k - t_c); dlogits written coalesced.
// HBM bytes: forward N*S*(4C + b_t), backward N*S*(8C + b_t), b_t = target bytes per voxel (1 / 8 for uint8 / int64 label maps,
// C / 4C for uint8 / fp32 C-channel targets).
#include "kernels.h"

namespace b200 {

namespace {

constexpr int kV = 128;             // voxels per tile
constexpr int kThreads = 128;       // one thread per voxel of a tile in the per-voxel phases
constexpr int kP = kV + 1;          // row pitch (floats) of the staged [C][kV] tiles: conflict-free column and row walks
constexpr int kSMs = 132;           // H100 SXM; with the shared-memory size it fixes the forward grid, hence the slot count
constexpr int kSmemPerSM = 228 * 1024;   // shared memory per SM; every resident block also takes kSmemReserved of it
constexpr int kSmemReserved = 1024;

__device__ __forceinline__ void cp_async4(float* dst, const float* src, bool valid) {
  const unsigned d = static_cast<unsigned>(__cvta_generic_to_shared(dst));
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(src), "r"(valid ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + __expf(-x)); }

__device__ __forceinline__ double warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

size_t tile_smem(int C, int kind) {
  size_t b = sizeof(double) * kThreads * 3 + sizeof(float) * (size_t)C * kP;   // reduction buffer + logits tile
  if (kind >= T_ONEHOT_U8) b += sizeof(float) * (size_t)C * kP;                 // target tile
  return b + sizeof(int) * kV + sizeof(float) * kV;                              // labels, 1 / sum of exponentials
}

// Blocks per sample: a whole number of resident waves on the H100, capped by the tiles.  A function of the shape alone.
int grid_x(int N, int C, long long S, int kind) {
  const long long tiles = (S + kV - 1) / kV;
  int per_sm = (int)(kSmemPerSM / (tile_smem(C, kind) + kSmemReserved));
  if (per_sm > 2048 / kThreads) per_sm = 2048 / kThreads;
  if (per_sm < 1) per_sm = 1;
  long long g = ((long long)kSMs * per_sm + N - 1) / N;
  if (g > tiles) g = tiles;
  return (int)(g < 1 ? 1 : g);
}

// Stage logits (and a C-channel target) of tile [s0, s0 + kV) of sample n; voxels past S read as zero, labels as -1.
template <int TK>
__device__ __forceinline__ void stage_tile(const float* __restrict__ xn, const void* __restrict__ tgt, int n, int C, long long S,
                                           long long s0, int nv, float* xs, float* ts, int* lab) {
  for (int i = threadIdx.x; i < C * kV; i += kThreads) {
    const int c = i / kV, v = i % kV;
    const bool ok = v < nv;
    cp_async4(xs + c * kP + v, xn + (ok ? (long long)c * S + s0 + v : 0), ok);
  }
  if (TK == T_SOFT_F32) {
    const float* tn = static_cast<const float*>(tgt) + (long long)n * C * S;
    for (int i = threadIdx.x; i < C * kV; i += kThreads) {
      const int c = i / kV, v = i % kV;
      const bool ok = v < nv;
      cp_async4(ts + c * kP + v, tn + (ok ? (long long)c * S + s0 + v : 0), ok);
    }
  } else if (TK == T_ONEHOT_U8) {
    const uint8_t* tn = static_cast<const uint8_t*>(tgt) + (long long)n * C * S;
#pragma unroll 4
    for (int i = threadIdx.x; i < C * kV; i += kThreads) {
      const int c = i / kV, v = i % kV;
      ts[c * kP + v] = v < nv ? (float)__ldg(tn + (long long)c * S + s0 + v) : 0.f;
    }
  } else {
    const int v = threadIdx.x;
    long long l = -1;
    if (v < nv) {
      l = TK == T_LABEL_U8 ? (long long)__ldg(static_cast<const uint8_t*>(tgt) + (long long)n * S + s0 + v)
                           : __ldg(reinterpret_cast<const long long*>(tgt) + (long long)n * S + s0 + v);
    }
    lab[v] = (l >= 0 && l < C) ? (int)l : -1;
  }
  cp_async_wait_all();
  __syncthreads();
}

struct Smem {
  double* red;
  float *xs, *ts, *inv;
  int* lab;
};
__device__ __forceinline__ Smem carve(unsigned char* base, int C, int kind) {
  Smem s;
  s.red = reinterpret_cast<double*>(base);
  s.xs = reinterpret_cast<float*>(s.red + kThreads * 3);
  s.ts = s.xs + C * kP;
  s.lab = reinterpret_cast<int*>(s.ts + (kind >= T_ONEHOT_U8 ? C * kP : 0));
  s.inv = reinterpret_cast<float*>(s.lab + kV);
  return s;
}

// grid (grid_x, N).  part [N][C][slots][3] (I, P, T), ce_part [N][slots] (zero without with_ce)
template <int TK, int ACT>
__global__ void __launch_bounds__(kThreads) k_dice_ce_fwd(const float* __restrict__ x, const void* __restrict__ tgt, int C, long long S,
                                                          int squared, int with_ce, double* __restrict__ part,
                                                          double* __restrict__ ce_part) {
  extern __shared__ __align__(16) unsigned char smem[];
  const Smem sm = carve(smem, C, TK);
  const int n = blockIdx.y, tid = threadIdx.x, slots = gridDim.x;
  const float* xn = x + (long long)n * C * S;
  const long long tiles = (S + kV - 1) / kV;
  const int K = kThreads / C, c = tid % C, slice = tid / C;   // phase B: thread (c, slice) walks voxels slice, slice + K, ...
  double aI = 0, aP = 0, aT = 0, ace = 0;
  for (long long tile = blockIdx.x; tile < tiles; tile += slots) {
    const long long s0 = tile * kV;
    const int nv = (int)(S - s0 < kV ? S - s0 : kV);
    stage_tile<TK>(xn, tgt, n, C, S, s0, nv, sm.xs, sm.ts, sm.lab);
    // phase A: one voxel per thread -- softmax statistics and the CE term
    if ((with_ce || ACT == A_SOFTMAX) && tid < nv) {
      const int v = tid;
      float ce;
      if (C == 1) {
        const float xv = sm.xs[v], t = sm.ts[v];
        ce = fmaxf(xv, 0.f) - xv * t + log1pf(__expf(-fabsf(xv)));
      } else {
        float m = -INFINITY;
        for (int k = 0; k < C; ++k) m = fmaxf(m, sm.xs[k * kP + v]);
        const int l = TK < T_ONEHOT_U8 ? sm.lab[v] : -1;
        const float xl = l >= 0 ? sm.xs[l * kP + v] : 0.f;
        float sum = 0.f, tx = 0.f, tsum = 0.f;
        for (int k = 0; k < C; ++k) {
          const float xv = sm.xs[k * kP + v];
          const float e = __expf(xv - m);
          sum += e;
          if (ACT == A_SOFTMAX) sm.xs[k * kP + v] = e;
          if (TK >= T_ONEHOT_U8) {
            const float t = sm.ts[k * kP + v];
            tx += t * xv;
            tsum += t;
          }
        }
        const float lse = m + logf(sum);
        if (ACT == A_SOFTMAX) sm.inv[v] = 1.f / sum;
        ce = TK >= T_ONEHOT_U8 ? lse * tsum - tx : (l >= 0 ? lse - xl : 0.f);
      }
      ace += ce;
    }
    __syncthreads();
    // phase B: channel c's Dice sums over this thread's slice of the tile
    if (slice < K) {
      float I[2] = {0.f, 0.f}, P[2] = {0.f, 0.f}, T[2] = {0.f, 0.f};   // two interleaved chains: voxels v and v + K
      auto acc = [&](int v, int j) {
        const float r = sm.xs[c * kP + v];
        const float p = ACT == A_SOFTMAX ? r * sm.inv[v] : ACT == A_SIGMOID ? sigm(r) : r;
        const float t = TK >= T_ONEHOT_U8 ? sm.ts[c * kP + v] : (sm.lab[v] == c ? 1.f : 0.f);
        I[j] += p * t;
        P[j] += squared ? p * p : p;
        T[j] += squared ? t * t : t;
      };
      int v = slice;
      for (; v + K < nv; v += 2 * K) { acc(v, 0); acc(v + K, 1); }
      if (v < nv) acc(v, 0);
      aI += I[0] + I[1]; aP += P[0] + P[1]; aT += T[0] + T[1];
    }
    __syncthreads();
  }
  // Dice sums: slices of a channel added in slice order; CE: a fixed-order block sum (warp trees, then the warps in order)
  __shared__ double sh_ce[kThreads / 32];
  sm.red[tid * 3 + 0] = aI; sm.red[tid * 3 + 1] = aP; sm.red[tid * 3 + 2] = aT;
  const double wce = warp_sum(ace);
  if ((tid & 31) == 0) sh_ce[tid >> 5] = wce;
  __syncthreads();
  if (tid < C) {
    double s[3] = {0, 0, 0};
    for (int k = 0; k < K; ++k)
      for (int j = 0; j < 3; ++j) s[j] += sm.red[(k * C + tid) * 3 + j];
    double* o = part + (((long long)n * C + tid) * slots + blockIdx.x) * 3;
    o[0] = s[0]; o[1] = s[1]; o[2] = s[2];
  }
  if (tid == 0) {
    double t = 0;
    for (int w = 0; w < kThreads / 32; ++w) t += sh_ce[w];
    ce_part[(long long)n * slots + blockIdx.x] = t;
  }
}

// one warp per (n, c) triple and per sample's CE: sums [N][C][3], ce [N]
__global__ void k_dice_ce_reduce(const double* __restrict__ part, const double* __restrict__ ce_part, int N, int C, int slots,
                                 double* __restrict__ sums, double* __restrict__ ce) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w < N * C) {
    const double* p = part + (long long)w * slots * 3;
    double a[3] = {0, 0, 0};
    for (int k = lane; k < slots; k += 32)
      for (int j = 0; j < 3; ++j) a[j] += p[k * 3 + j];
    for (int j = 0; j < 3; ++j) {
      const double r = warp_sum(a[j]);
      if (lane == 0) sums[(long long)w * 3 + j] = r;
    }
  } else if (w < N * C + N) {
    const int n = w - N * C;
    double a = 0;
    for (int k = lane; k < slots; k += 32) a += ce_part[(long long)n * slots + k];
    a = warp_sum(a);
    if (lane == 0) ce[n] = a;
  }
}

// grid (grid_x, N); one voxel per thread
template <int TK, int ACT>
__global__ void __launch_bounds__(kThreads) k_dice_ce_bwd(const float* __restrict__ x, const void* __restrict__ tgt, int C, long long S,
                                                          int squared, int with_ce, double ce_scale, const double* __restrict__ coef,
                                                          const float* __restrict__ grad_out, float* __restrict__ dx) {
  extern __shared__ __align__(16) unsigned char smem[];
  const Smem sm = carve(smem, C, TK);
  float* a = reinterpret_cast<float*>(sm.red);      // [C] dF/dI and [C] dF/dP coefficients of sample n, times grad_out
  float* b = a + C;
  const int n = blockIdx.y, v = threadIdx.x;
  const float go = *grad_out;
  for (int c = v; c < C; c += kThreads) {
    a[c] = (float)(coef[((long long)n * C + c) * 2] * go);
    b[c] = (float)(coef[((long long)n * C + c) * 2 + 1] * go);
  }
  const float cg = (float)(ce_scale * go);
  const float* xn = x + (long long)n * C * S;
  float* dxn = dx + (long long)n * C * S;
  const long long tiles = (S + kV - 1) / kV;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long s0 = tile * kV;
    const int nv = (int)(S - s0 < kV ? S - s0 : kV);
    stage_tile<TK>(xn, tgt, n, C, S, s0, nv, sm.xs, sm.ts, sm.lab);   // its barrier also publishes a / b
    if (v < nv) {
      float* o = dxn + s0 + v;
      if (C == 1) {
        const float xv = sm.xs[v], t = sm.ts[v];
        const float q = sigm(xv);
        const float p = ACT == A_SIGMOID ? q : xv;
        const float g = a[0] * t + b[0] * (squared ? 2.f * p : 1.f);
        *o = (ACT == A_SIGMOID ? g * p * (1.f - p) : g) + cg * (q - t);
      } else {
        const int l = TK < T_ONEHOT_U8 ? sm.lab[v] : -1;
        float m = -INFINITY, inv = 0.f, tsum = 0.f;
        if (with_ce || ACT == A_SOFTMAX) {
          for (int k = 0; k < C; ++k) m = fmaxf(m, sm.xs[k * kP + v]);
          float sum = 0.f;
          for (int k = 0; k < C; ++k) {
            const float e = __expf(sm.xs[k * kP + v] - m);
            sum += e;
            if (ACT == A_SOFTMAX) sm.xs[k * kP + v] = e;
            if (TK >= T_ONEHOT_U8) tsum += sm.ts[k * kP + v];
          }
          inv = 1.f / sum;
        }
        if (TK < T_ONEHOT_U8) tsum = l >= 0 ? 1.f : 0.f;
        if (ACT == A_SOFTMAX) {
          float s = 0.f;
          for (int k = 0; k < C; ++k) {
            const float p = sm.xs[k * kP + v] * inv;
            const float t = TK >= T_ONEHOT_U8 ? sm.ts[k * kP + v] : (k == l ? 1.f : 0.f);
            s += p * (a[k] * t + b[k] * (squared ? 2.f * p : 1.f));
          }
          for (int k = 0; k < C; ++k) {
            const float p = sm.xs[k * kP + v] * inv;
            const float t = TK >= T_ONEHOT_U8 ? sm.ts[k * kP + v] : (k == l ? 1.f : 0.f);
            const float g = a[k] * t + b[k] * (squared ? 2.f * p : 1.f);
            o[(long long)k * S] = p * (g - s) + cg * (p * tsum - t);
          }
        } else {
          for (int k = 0; k < C; ++k) {
            const float xv = sm.xs[k * kP + v];
            const float p = ACT == A_SIGMOID ? sigm(xv) : xv;
            const float t = TK >= T_ONEHOT_U8 ? sm.ts[k * kP + v] : (k == l ? 1.f : 0.f);
            const float g = a[k] * t + b[k] * (squared ? 2.f * p : 1.f);
            const float dd = ACT == A_SIGMOID ? g * p * (1.f - p) : g;
            o[(long long)k * S] = with_ce ? dd + cg * (__expf(xv - m) * inv * tsum - t) : dd;
          }
        }
      }
    }
    __syncthreads();
  }
}

struct Shape {
  int N, C, kind, act, slots;
  long long S;
};

int check_shape(const DiceCEDesc& d, int N, int C, long long S, Shape* sh) {
  B200_TRY(check_dice_desc(d, N, C, S, "dice_ce"));
  B200_REQUIRE(C <= 128, E_UNSUPPORTED, "dice_ce: %d channels (at most 128)", C);
  sh->N = N; sh->C = C; sh->S = S; sh->kind = d.target_kind; sh->act = d.act;
  if (C == 1) {
    // one channel: softmax and the label-map expansion do not apply (MONAI ignores them); a uint8 map is the uint8 target itself
    B200_REQUIRE(d.target_kind != T_LABEL_I64, E_UNSUPPORTED, "dice_ce: one channel with an int64 target (pass uint8 or fp32)");
    if (sh->kind == T_LABEL_U8) sh->kind = T_ONEHOT_U8;
    if (sh->act == A_SOFTMAX) sh->act = A_NONE;
  }
  sh->slots = grid_x(N, C, S, sh->kind);
  return OK;
}

struct Scratch {
  double *sums, *ce, *coef, *part, *ce_part;
};
Scratch carve_scratch(void* base, const Shape& s) {
  Scratch r;
  r.sums = static_cast<double*>(base);
  r.ce = r.sums + (size_t)s.N * s.C * 3;
  r.coef = r.ce + s.N;
  r.part = r.coef + (size_t)s.N * s.C * 2;
  r.ce_part = r.part + (size_t)s.N * s.C * s.slots * 3;
  return r;
}

template <typename K>
int set_smem(K kernel, size_t bytes) {
  if (bytes > 48 * 1024) B200_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return OK;
}

#define B200_DICE_CE_SWITCH(M)                                                   \
  switch (sh.kind * 3 + sh.act) {                                                \
    case 0: M(0, 0); break; case 1: M(0, 1); break; case 2: M(0, 2); break;      \
    case 3: M(1, 0); break; case 4: M(1, 1); break; case 5: M(1, 2); break;      \
    case 6: M(2, 0); break; case 7: M(2, 1); break; case 8: M(2, 2); break;      \
    case 9: M(3, 0); break; case 10: M(3, 1); break; default: M(3, 2); break;    \
  }

}  // namespace

size_t dice_ce_scratch_bytes(const DiceCEDesc& d, int N, int C, long long S) {
  Shape sh;
  if (check_shape(d, N, C, S, &sh) != OK) return 0;
  return sizeof(double) * ((size_t)sh.N * sh.C * (3 + 2 + 3 * (size_t)sh.slots) + (size_t)sh.N * (1 + sh.slots));
}

int launch_dice_ce_fwd(const DiceCEDesc& d, const float* logits, const void* target, int N, int C, long long S, void* scratch,
                       float* loss, cudaStream_t st) {
  Shape sh;
  B200_TRY(check_shape(d, N, C, S, &sh));
  const Scratch s = carve_scratch(scratch, sh);
  const size_t smem = tile_smem(sh.C, sh.kind);
  const dim3 grid(sh.slots, N);
  const int with_ce = d.lambda_ce != 0.f;
#define B200_FWD(tk, ac)                                                                                                \
  B200_TRY(set_smem(k_dice_ce_fwd<tk, ac>, smem));                                                                      \
  k_dice_ce_fwd<tk, ac><<<grid, kThreads, smem, st>>>(logits, target, C, S, d.squared_pred, with_ce, s.part, s.ce_part);
  B200_DICE_CE_SWITCH(B200_FWD)
#undef B200_FWD
  B200_CHECK_CUDA(cudaGetLastError());
  const int warps = N * C + N;
  k_dice_ce_reduce<<<(warps + 7) / 8, 256, 0, st>>>(s.part, s.ce_part, N, C, sh.slots, s.sums, s.ce);
  B200_CHECK_CUDA(cudaGetLastError());
  return launch_dice_finalize(d, s.sums, s.ce, N, C, S, s.coef, loss, st);
}

int launch_dice_ce_bwd(const DiceCEDesc& d, const float* logits, const void* target, int N, int C, long long S, const void* scratch,
                       const float* grad_out, float* dlogits, cudaStream_t st) {
  Shape sh;
  B200_TRY(check_shape(d, N, C, S, &sh));
  const Scratch s = carve_scratch(const_cast<void*>(scratch), sh);
  const size_t smem = tile_smem(sh.C, sh.kind);
  const dim3 grid(sh.slots, N);
  const int with_ce = d.lambda_ce != 0.f;
  const double ce_scale = d.lambda_ce * (d.reduction == 0 ? 1.0 / ((double)N * S) : 1.0);
#define B200_BWD(tk, ac)                                                                                                 \
  B200_TRY(set_smem(k_dice_ce_bwd<tk, ac>, smem));                                                                       \
  k_dice_ce_bwd<tk, ac><<<grid, kThreads, smem, st>>>(logits, target, C, S, d.squared_pred, with_ce, ce_scale, s.coef,   \
                                                      grad_out, dlogits);
  B200_DICE_CE_SWITCH(B200_BWD)
#undef B200_BWD
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

#undef B200_DICE_CE_SWITCH

}  // namespace b200
