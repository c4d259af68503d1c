// Bandwidth-shaped rewrites of four small kernels that per-launch timing showed far from the HBM roofline:
//   * weight packing / gradient unpacking: shared-memory tiled transposes (the straightforward gather read fp32 weights
//     with a 108-byte stride between neighbouring threads)
//   * trilinear x2 adjoint: the 4x4x4 neighbourhood of every output voxel comes from a shared-memory tile instead of 64
//     L2 reads per thread (8x read amplification -> 2.3x)
//   * weight gradient of a 1x1x1 convolution with <= 16 input channels (the first residual block's `sample`,
//     myronenko.py:42-45 with 4 input channels): a register-tile outer product at the streaming rate; the tensor-core
//     path spends a 128-row MMA tile on 8 useful rows
// All keep the interfaces of the kernels they replace (kernels.h); B200UNET_OLD_SMALL_OPS=1 selects the round-1 versions.
#include <cstdlib>
#include "kernels.h"
#include "ptx.cuh"

namespace b200 {

static bool old_small_ops() {
  static const bool v = getenv("B200UNET_OLD_SMALL_OPS") != nullptr;
  return v;
}

__device__ __forceinline__ void ld8(const bf16* hi, const bf16* lo, long long off, float (&v)[8]) {
  const uint4 a = *reinterpret_cast<const uint4*>(hi + off);
  v[0] = bf16_lo_to_f(a.x); v[1] = bf16_hi_to_f(a.x); v[2] = bf16_lo_to_f(a.y); v[3] = bf16_hi_to_f(a.y);
  v[4] = bf16_lo_to_f(a.z); v[5] = bf16_hi_to_f(a.z); v[6] = bf16_lo_to_f(a.w); v[7] = bf16_hi_to_f(a.w);
  if (lo) {
    const uint4 b = *reinterpret_cast<const uint4*>(lo + off);
    v[0] += bf16_lo_to_f(b.x); v[1] += bf16_hi_to_f(b.x); v[2] += bf16_lo_to_f(b.y); v[3] += bf16_hi_to_f(b.y);
    v[4] += bf16_lo_to_f(b.z); v[5] += bf16_hi_to_f(b.z); v[6] += bf16_lo_to_f(b.w); v[7] += bf16_hi_to_f(b.w);
  }
}
__device__ __forceinline__ void st8(bf16* hi, bf16* lo, long long off, const float (&v)[8]) {
  uint4 a;
  a.x = pack_bf16x2(v[0], v[1]); a.y = pack_bf16x2(v[2], v[3]); a.z = pack_bf16x2(v[4], v[5]); a.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(hi + off) = a;
  if (lo) {
    uint4 b;
    b.x = pack_bf16x2(v[0] - bf16_lo_to_f(a.x), v[1] - bf16_hi_to_f(a.x));
    b.y = pack_bf16x2(v[2] - bf16_lo_to_f(a.y), v[3] - bf16_hi_to_f(a.y));
    b.z = pack_bf16x2(v[4] - bf16_lo_to_f(a.z), v[5] - bf16_hi_to_f(a.z));
    b.w = pack_bf16x2(v[6] - bf16_lo_to_f(a.w), v[7] - bf16_hi_to_f(a.w));
    *reinterpret_cast<uint4*>(lo + off) = b;
  }
}

// ------------------------------------------------------------------------------------------------ weight pack (tiled)
// One block transposes 16 (co) x 16 (ci) x T (taps) elements through shared memory: the fp32 source is read in runs of
// 16*T contiguous floats, both packed layouts are written in 32-byte (16 x bf16) segments.  Job modes as in kernels.h.
constexpr int PT = 16;        // tile edge along co and ci
constexpr int PTT = 29;       // padded tap pitch (27 taps; odd pitch: conflict-free column reads)

// TC: compile-time tap count (27, 8, 1) so that the index divisions fold into multiplies; 0 = runtime j.T
template <int TC>
__device__ __forceinline__ void pack_job_tiled(float (&tile)[PT][PT + 1][PTT], const PackJob& j, const float* __restrict__ w,
                                               bf16* __restrict__ hi, bf16* __restrict__ lo) {
  const int T = TC ? TC : j.T;
  const bool tsrc = j.mode >= 2;                       // ConvTranspose3d weight [Ci][Co][T]
  const bool flip = j.mode == 1 || j.mode == 2;
  const bool co_inner = j.mode == 1 || j.mode == 3;    // data-gradient layout [T][Cip][Cop]
  const int nco = (j.Cop + PT - 1) / PT, nci = (j.Cip + PT - 1) / PT;
  for (int tl = blockIdx.x; tl < nco * nci; tl += gridDim.x) {
    const int co0 = (tl / nci) * PT, ci0 = (tl % nci) * PT;
    __syncthreads();   // the previous tile has been written out
    for (int idx = threadIdx.x; idx < PT * PT * T; idx += blockDim.x) {
      const int o = idx / (PT * T), rem = idx % (PT * T), i = rem / T, t = rem % T;
      float v = 0.f;
      if (!tsrc) {   // outer = co, inner run = (ci, t)
        const int co = co0 + o, ci = ci0 + i;
        if (co < j.Co && ci < j.Ci) v = w[((long long)co * j.Ci + ci) * T + t];
        tile[o][i][t] = v;
      } else {       // outer = ci, inner run = (co, t)
        const int ci = ci0 + o, co = co0 + i;
        if (co < j.Co && ci < j.Ci) v = w[((long long)ci * j.Co + co) * T + t];
        tile[i][o][t] = v;
      }
    }
    __syncthreads();
    // write phase: one 16-byte store (8 bf16 along the destination's inner channel axis) per thread and step; padded channel
    // counts are multiples of 8 and the tile origin of 16, so a chunk is either wholly inside the padded extent or skipped
    for (int idx = threadIdx.x; idx < PT * 2 * T; idx += blockDim.x) {
      const int t = idx / (PT * 2), rem = idx % (PT * 2), outer = rem >> 1, half = (rem & 1) * 8;
      const int ts = flip ? T - 1 - t : t;
      float v[8];
      long long dst;
      if (!co_inner) {   // [T][Cop][Cip]: outer = co, chunk along ci
        if (co0 + outer >= j.Cop || ci0 + half >= j.Cip) continue;
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = tile[outer][half + q][ts];
        dst = ((long long)t * j.Cop + co0 + outer) * j.Cip + ci0 + half;
      } else {           // [T][Cip][Cop]: outer = ci, chunk along co
        if (ci0 + outer >= j.Cip || co0 + half >= j.Cop) continue;
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = tile[half + q][outer][ts];
        dst = ((long long)t * j.Cip + ci0 + outer) * j.Cop + co0 + half;
      }
      uint4 a;
      a.x = pack_bf16x2(v[0], v[1]); a.y = pack_bf16x2(v[2], v[3]); a.z = pack_bf16x2(v[4], v[5]); a.w = pack_bf16x2(v[6], v[7]);
      *reinterpret_cast<uint4*>(hi + dst) = a;
      if (lo) {
        uint4 b;
        b.x = pack_bf16x2(v[0] - bf16_lo_to_f(a.x), v[1] - bf16_hi_to_f(a.x));
        b.y = pack_bf16x2(v[2] - bf16_lo_to_f(a.y), v[3] - bf16_hi_to_f(a.y));
        b.z = pack_bf16x2(v[4] - bf16_lo_to_f(a.z), v[5] - bf16_hi_to_f(a.z));
        b.w = pack_bf16x2(v[6] - bf16_lo_to_f(a.w), v[7] - bf16_hi_to_f(a.w));
        *reinterpret_cast<uint4*>(lo + dst) = b;
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_pack_all_tiled(PtrTable params, const PackJob* __restrict__ jobs, uint8_t* __restrict__ ws,
                                                       int split) {
  __shared__ float tile[PT][PT + 1][PTT];   // odd (ci) pitch: both store orders read (nearly) conflict-free
  const PackJob j = jobs[blockIdx.y];
  const float* __restrict__ w = reinterpret_cast<const float*>(params.p[j.pidx]);
  bf16* hi = reinterpret_cast<bf16*>(ws + j.off_hi);
  bf16* lo = split ? reinterpret_cast<bf16*>(ws + j.off_lo) : nullptr;
  if (j.T == 27) pack_job_tiled<27>(tile, j, w, hi, lo);
  else if (j.T == 1) pack_job_tiled<1>(tile, j, w, hi, lo);
  else if (j.T == 8) pack_job_tiled<8>(tile, j, w, hi, lo);
  else pack_job_tiled<0>(tile, j, w, hi, lo);
}

template <int TC>
__device__ __forceinline__ void unpack_job_tiled(float (&tile)[PT][PT + 1][PTT], const PackJob& j, const float* __restrict__ g,
                                                 float* __restrict__ out) {
  const int T = TC ? TC : j.T;
  const bool tdst = j.mode == 2;   // ConvTranspose3d gradient layout [Ci][Co][T], taps flipped back
  const int nco = (j.Co + PT - 1) / PT, nci = (j.Ci + PT - 1) / PT;
  for (int tl = blockIdx.x; tl < nco * nci; tl += gridDim.x) {
    const int co0 = (tl / nci) * PT, ci0 = (tl % nci) * PT;
    __syncthreads();
    for (int idx = threadIdx.x; idx < PT * PT * T; idx += blockDim.x) {
      const int t = idx / (PT * PT), rem = idx % (PT * PT), cil = rem / PT, col = rem % PT;
      float v = 0.f;
      if (co0 + col < j.Co && ci0 + cil < j.Ci) v = g[((long long)t * j.Cip + ci0 + cil) * j.Cop + co0 + col];
      tile[col][cil][t] = v;
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < PT * PT * T; idx += blockDim.x) {
      const int o = idx / (PT * T), rem = idx % (PT * T), i = rem / T, t = rem % T;
      if (!tdst) {
        const int co = co0 + o, ci = ci0 + i;
        if (co < j.Co && ci < j.Ci) out[((long long)co * j.Ci + ci) * T + t] = tile[o][i][t];
      } else {
        const int ci = ci0 + o, co = co0 + i;
        if (co < j.Co && ci < j.Ci) out[((long long)ci * j.Co + co) * T + t] = tile[i][o][T - 1 - t];
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_unpack_all_tiled(PtrTable grads, const PackJob* __restrict__ jobs,
                                                         const uint8_t* __restrict__ ws) {
  __shared__ float tile[PT][PT + 1][PTT];
  const PackJob j = jobs[blockIdx.y];
  float* __restrict__ out = const_cast<float*>(reinterpret_cast<const float*>(grads.p[j.pidx]));
  const float* __restrict__ g = reinterpret_cast<const float*>(ws + j.off_hi);   // fp32 accumulator [T][Cip][Cop]
  if (j.T == 27) unpack_job_tiled<27>(tile, j, g, out);
  else if (j.T == 1) unpack_job_tiled<1>(tile, j, g, out);
  else if (j.T == 8) unpack_job_tiled<8>(tile, j, g, out);
  else unpack_job_tiled<0>(tile, j, g, out);
}

int launch_pack_all_tiled(const PtrTable& params, const PackJob* jobs_dev, int njobs, uint8_t* ws, bool split, cudaStream_t st) {
  if (njobs == 0) return OK;
  k_pack_all_tiled<<<dim3(256, njobs), 256, 0, st>>>(params, jobs_dev, ws, split ? 1 : 0);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

int launch_unpack_all_tiled(const PtrTable& grads, const PackJob* jobs_dev, int njobs, const uint8_t* ws, cudaStream_t st) {
  if (njobs == 0) return OK;
  k_unpack_all_tiled<<<dim3(256, njobs), 256, 0, st>>>(grads, jobs_dev, ws);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

bool use_tiled_pack() { return !old_small_ops(); }

// ------------------------------------------------------------------------------------------------ trilinear x2 adjoint (tiled)
// dx[k] = .25 dy[2k-1] + .75 dy[2k] + .75 dy[2k+1] + .25 dy[2k+2] per axis, where a position outside [0, 2n) hands its
// weight to the clamped neighbour (out[0] and out[2n-1] of the forward read x[0] / x[n-1] twice).  A block owns a
// 2 x 4 x 4 tile of dx and CT = 32 channels: the 6 x 10 x 10 dy neighbourhood is staged in shared memory once.
constexpr int UD = 2, UH = 4, UW = 4, UCT = 32;
constexpr int URD = 2 * UD + 2, URH = 2 * UH + 2, URW = 2 * UW + 2;

__device__ __forceinline__ void up_adj_w(int k, int n, float (&w)[4]) {
  w[0] = 0.25f; w[1] = 0.75f; w[2] = 0.75f; w[3] = 0.25f;
  if (k == 0) { w[0] = 0.f; w[1] = 1.0f; }
  if (k == n - 1) { w[3] = 0.f; w[2] = 1.0f; }
}

template <bool SPLIT>
__global__ void __launch_bounds__(UD * UH * UW * (UCT / 8)) k_upsample2x_bwd_tiled(Act dy, Act dx, int tiles_w, int tiles_h, int tiles_d,
                                                                               int cgroups) {
  extern __shared__ uint4 s_up[];
  uint4* s_hi = s_up;
  uint4* s_lo = s_up + URD * URH * URW * (UCT / 8);   // only present in split precision
  int t = blockIdx.x;
  const int cg = t % cgroups; t /= cgroups;
  const int wt = t % tiles_w; t /= tiles_w;
  const int ht = t % tiles_h; t /= tiles_h;
  const int dt = t % tiles_d;
  const int n = t / tiles_d;
  const int w0 = wt * UW, h0 = ht * UH, d0 = dt * UD, c0 = cg * UCT;
  constexpr bool split = SPLIT;
  constexpr int NCH = UCT / 8;
  for (int i = threadIdx.x; i < URD * URH * URW * NCH; i += blockDim.x) {
    const int ch = i % NCH;
    int r = i / NCH;
    const int lw = r % URW; r /= URW;
    const int lh = r % URH;
    const int ld_ = r / URH;
    const int gw = 2 * w0 - 1 + lw, gh = 2 * h0 - 1 + lh, gd = 2 * d0 - 1 + ld_;
    uint4 a = make_uint4(0u, 0u, 0u, 0u), b = a;
    if (gw >= 0 && gw < dy.W && gh >= 0 && gh < dy.H && gd >= 0 && gd < dy.D && c0 + ch * 8 < dy.C) {
      const long long off = ((((long long)n * dy.D + gd) * dy.H + gh) * dy.W + gw) * dy.ld + c0 + ch * 8;
      a = *reinterpret_cast<const uint4*>(dy.hi + off);
      if (split) b = *reinterpret_cast<const uint4*>(dy.lo + off);
    }
    s_hi[i] = a;
    if (split) s_lo[i] = b;
  }
  __syncthreads();
  const int ch = threadIdx.x % NCH;
  int v = threadIdx.x / NCH;
  const int lw = v % UW; v /= UW;
  const int lh = v % UH;
  const int ldd = v / UH;
  const int w = w0 + lw, h = h0 + lh, d = d0 + ldd;
  if (w >= dx.W || h >= dx.H || d >= dx.D || c0 + ch * 8 >= dx.C) return;
  float wd[4], wh[4], ww[4];
  up_adj_w(d, dx.D, wd); up_adj_w(h, dx.H, wh); up_adj_w(w, dx.W, ww);
  float o[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = 0.f;
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const float wab = wd[a] * wh[b];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int si = (((2 * ldd + a) * URH + 2 * lh + b) * URW + 2 * lw + c) * NCH + ch;
        const float wt_ = wab * ww[c];
        const uint4 p = s_hi[si];
        o[0] = fmaf(wt_, bf16_lo_to_f(p.x), o[0]); o[1] = fmaf(wt_, bf16_hi_to_f(p.x), o[1]);
        o[2] = fmaf(wt_, bf16_lo_to_f(p.y), o[2]); o[3] = fmaf(wt_, bf16_hi_to_f(p.y), o[3]);
        o[4] = fmaf(wt_, bf16_lo_to_f(p.z), o[4]); o[5] = fmaf(wt_, bf16_hi_to_f(p.z), o[5]);
        o[6] = fmaf(wt_, bf16_lo_to_f(p.w), o[6]); o[7] = fmaf(wt_, bf16_hi_to_f(p.w), o[7]);
        if (split) {
          const uint4 q = s_lo[si];
          o[0] = fmaf(wt_, bf16_lo_to_f(q.x), o[0]); o[1] = fmaf(wt_, bf16_hi_to_f(q.x), o[1]);
          o[2] = fmaf(wt_, bf16_lo_to_f(q.y), o[2]); o[3] = fmaf(wt_, bf16_hi_to_f(q.y), o[3]);
          o[4] = fmaf(wt_, bf16_lo_to_f(q.z), o[4]); o[5] = fmaf(wt_, bf16_hi_to_f(q.z), o[5]);
          o[6] = fmaf(wt_, bf16_lo_to_f(q.w), o[6]); o[7] = fmaf(wt_, bf16_hi_to_f(q.w), o[7]);
        }
      }
    }
  st8(dx.hi, dx.lo, ((((long long)n * dx.D + d) * dx.H + h) * dx.W + w) * dx.ld + c0 + ch * 8, o);
}

bool use_tiled_upsample_bwd() {
  // slower than the L1-cached gather version where it was first measured -> kept as an opt-in experiment
  static const bool v = getenv("B200UNET_TILED_UPSAMPLE_BWD") != nullptr;
  return v;
}

int launch_upsample2x_bwd_tiled(const Act& dy, const Act& dx, cudaStream_t st) {
  B200_REQUIRE(dx.C % 8 == 0 && dy.C == dx.C, E_INVALID, "upsample_bwd: channel mismatch");
  B200_REQUIRE(dy.D == 2 * dx.D && dy.H == 2 * dx.H && dy.W == 2 * dx.W, E_UNSUPPORTED, "upsample_bwd: not 2x");
  const int tw = ceil_div(dx.W, UW), th = ceil_div(dx.H, UH), td = ceil_div(dx.D, UD), cgs = ceil_div(dx.C, UCT);
  const long long blocks = (long long)dx.N * td * th * tw * cgs;
  B200_REQUIRE(blocks < (1LL << 31), E_UNSUPPORTED, "upsample_bwd: volume too large");
  const int tile_bytes = URD * URH * URW * (UCT / 8) * (int)sizeof(uint4);
  if (dy.lo) {
    B200_REQUIRE(dx.lo != nullptr, E_INVALID, "upsample_bwd: split input needs a split output");
    static bool attr_set[64] = {false};
    int dev = 0;
    B200_CHECK_CUDA(cudaGetDevice(&dev));
    if (dev < 64 && !attr_set[dev]) {
      B200_CHECK_CUDA(cudaFuncSetAttribute(k_upsample2x_bwd_tiled<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * tile_bytes));
      attr_set[dev] = true;
    }
    k_upsample2x_bwd_tiled<true><<<(unsigned)blocks, UD * UH * UW * (UCT / 8), 2 * tile_bytes, st>>>(dy, dx, tw, th, td, cgs);
  } else {
    k_upsample2x_bwd_tiled<false><<<(unsigned)blocks, UD * UH * UW * (UCT / 8), tile_bytes, st>>>(dy, dx, tw, th, td, cgs);
  }
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// ------------------------------------------------------------------------------------------------ 1x1x1 weight gradient, narrow input
// dW[ci][co] += sum_v a[v][ci] * dy[v][co]   for Ci = 8 * CI8 <= 16.  Thread <-> (voxel slot, 8-channel chunk of dy): it keeps a
// (Ci x 8) fp32 tile of dW in registers over its whole grid-stride loop; reduced by warp shuffles over the lanes that share
// the chunk, shared-memory atomics across warps, then one global atomic per element per block.
template <int CI8>
__global__ void __launch_bounds__(256, CI8 == 1 ? 2 : 1) k_wgrad_1x1_narrow(Act a, Act dy, float* __restrict__ dw, int Cop) {
  extern __shared__ float s_dw[];   // [Ci][Co]
  const int Ci = CI8 * 8, Co = dy.C;
  for (int i = threadIdx.x; i < Ci * Co; i += blockDim.x) s_dw[i] = 0.f;
  __syncthreads();
  const int c8n = Co / 8;
  const int cy = threadIdx.x % c8n;
  const int vslot = threadIdx.x / c8n, vper = blockDim.x / c8n;
  float acc[CI8 * 8][8];
#pragma unroll
  for (int i = 0; i < CI8 * 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  const long long total = a.voxels();
  const long long stride = (long long)gridDim.x * vper;
  // UF voxels in flight per thread: all loads of an iteration are issued before the first FMA (one voxel per iteration left
  // the kernel latency-bound at ~1.3 TB/s)
  constexpr int UF = 2;
  for (long long v0 = (long long)blockIdx.x * vper + vslot; v0 < total; v0 += UF * stride) {
    uint4 gq[UF], xq[UF][CI8];
#pragma unroll
    for (int q = 0; q < UF; ++q) {
      const long long v = v0 + q * stride;
      if (v < total) {
        gq[q] = *reinterpret_cast<const uint4*>(dy.hi + v * dy.ld + cy * 8);
#pragma unroll
        for (int c = 0; c < CI8; ++c) xq[q][c] = *reinterpret_cast<const uint4*>(a.hi + v * a.ld + c * 8);
      } else {
        gq[q] = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int c = 0; c < CI8; ++c) xq[q][c] = make_uint4(0u, 0u, 0u, 0u);
      }
    }
#pragma unroll
    for (int q = 0; q < UF; ++q) {
      const long long v = v0 + q * stride;
      float g[8];
      g[0] = bf16_lo_to_f(gq[q].x); g[1] = bf16_hi_to_f(gq[q].x); g[2] = bf16_lo_to_f(gq[q].y); g[3] = bf16_hi_to_f(gq[q].y);
      g[4] = bf16_lo_to_f(gq[q].z); g[5] = bf16_hi_to_f(gq[q].z); g[6] = bf16_lo_to_f(gq[q].w); g[7] = bf16_hi_to_f(gq[q].w);
      if (dy.lo && v < total) {
        float gl[8];
        ld8(dy.lo, nullptr, v * dy.ld + cy * 8, gl);
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] += gl[j];
      }
#pragma unroll
      for (int c = 0; c < CI8; ++c) {
        float x[8];
        const uint4 xa = xq[q][c];
        x[0] = bf16_lo_to_f(xa.x); x[1] = bf16_hi_to_f(xa.x); x[2] = bf16_lo_to_f(xa.y); x[3] = bf16_hi_to_f(xa.y);
        x[4] = bf16_lo_to_f(xa.z); x[5] = bf16_hi_to_f(xa.z); x[6] = bf16_lo_to_f(xa.w); x[7] = bf16_hi_to_f(xa.w);
        if (a.lo && v < total) {
          float xl[8];
          ld8(a.lo, nullptr, v * a.ld + c * 8, xl);
#pragma unroll
          for (int j = 0; j < 8; ++j) x[j] += xl[j];
        }
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[c * 8 + i][j] = fmaf(x[i], g[j], acc[c * 8 + i][j]);
      }
    }
  }
  const bool pow2 = (c8n & (c8n - 1)) == 0 && c8n <= 32;   // then lanes l, l' share the chunk iff l % c8n == l' % c8n
#pragma unroll
  for (int i = 0; i < CI8 * 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float p = acc[i][j];
      if (pow2) {
        for (int off = 16; off >= c8n; off >>= 1) p += __shfl_xor_sync(0xffffffffu, p, off);
        if ((threadIdx.x & 31) < c8n) atomicAdd(&s_dw[i * Co + cy * 8 + j], p);
      } else {
        atomicAdd(&s_dw[i * Co + cy * 8 + j], p);
      }
    }
  __syncthreads();
  for (int i = threadIdx.x; i < Ci * Co; i += blockDim.x) atomicAdd(&dw[(long long)(i / Co) * Cop + (i % Co)], s_dw[i]);
}

bool wgrad_1x1_narrow_eligible(const WgradOp& op) {
  if (old_small_ops()) return false;
  return op.ksz == 1 && op.stride == 1 && op.a.C <= 16 && op.a.C % 8 == 0 && op.dy.C % 8 == 0 && op.dy.C <= 256 && !op.a.vD && !op.dy.vD &&
         256 % (op.dy.C / 8) == 0;
}

int launch_wgrad_1x1_narrow(const WgradOp& op, cudaStream_t st) {
  B200_REQUIRE(wgrad_1x1_narrow_eligible(op), E_UNSUPPORTED, "wgrad_1x1_narrow: shape not eligible");
  B200_REQUIRE(op.a.N == op.dy.N && op.a.D == op.dy.D && op.a.H == op.dy.H && op.a.W == op.dy.W, E_INVALID, "wgrad_1x1_narrow: shape mismatch");
  const int c8n = op.dy.C / 8;
  const int vper = 256 / c8n;
  const long long want = (op.a.voxels() + vper - 1) / vper;
  const int blocks = (int)(want < 132 * 6 ? (want > 0 ? want : 1) : 132 * 6);
  const size_t smem = (size_t)op.a.C * op.dy.C * sizeof(float);
  if (op.a.C == 8) k_wgrad_1x1_narrow<1><<<blocks, 256, smem, st>>>(op.a, op.dy, op.dw, op.Cop);
  else k_wgrad_1x1_narrow<2><<<blocks, 256, smem, st>>>(op.a, op.dy, op.dw, op.Cop);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

}  // namespace b200
