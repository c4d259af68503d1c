// Bandwidth-shaped kernels for small jobs that per-launch timing showed far from the HBM roofline in their straightforward form:
//   * weight packing / gradient unpacking: shared-memory tiled transposes (a gather reads the fp32 weights with a 108-byte
//     stride between neighbouring threads)
//   * weight gradient of a 1x1x1 convolution with <= 16 input channels (the first residual block's `sample`,
//     myronenko.py:42-45 with 4 input channels): a register-tile outer product at the streaming rate; the tensor-core
//     path spends a 128-row MMA tile on 8 useful rows
#include "kernels.h"
#include "ptx.cuh"

namespace b200 {

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
  const bool tsrc = j.mode >= PACK_T_FLIPPED;                           // ConvTranspose3d weight [Ci][Co][T]
  const bool flip = j.mode == PACK_DGRAD || j.mode == PACK_T_FLIPPED;
  const bool co_inner = j.mode == PACK_DGRAD || j.mode == PACK_T_DGRAD;   // data-gradient layout [T][Cip][Cop]
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
      store8(hi, lo, dst, v);
    }
  }
}

// the tap counts of 3x3x3, 1x1x1 and 2x2x2 weights at compile time
__device__ __forceinline__ void pack_job(float (&tile)[PT][PT + 1][PTT], const PackJob& j, const float* w, bf16* hi, bf16* lo) {
  if (j.T == 27) pack_job_tiled<27>(tile, j, w, hi, lo);
  else if (j.T == 1) pack_job_tiled<1>(tile, j, w, hi, lo);
  else if (j.T == 8) pack_job_tiled<8>(tile, j, w, hi, lo);
  else pack_job_tiled<0>(tile, j, w, hi, lo);
}

__global__ void __launch_bounds__(256) k_pack_all_tiled(PtrTable params, const PackJob* __restrict__ jobs, uint8_t* __restrict__ ws,
                                                       int split) {
  __shared__ float tile[PT][PT + 1][PTT];   // odd (ci) pitch: both store orders read (nearly) conflict-free
  const PackJob j = jobs[blockIdx.y];
  const float* __restrict__ w = reinterpret_cast<const float*>(params.p[j.pidx]);
  bf16* hi = reinterpret_cast<bf16*>(ws + j.off_hi);
  bf16* lo = split ? reinterpret_cast<bf16*>(ws + j.off_lo) : nullptr;
  pack_job(tile, j, w, hi, lo);
}

// one tensor (the per-tensor C ABI entry points)
__global__ void __launch_bounds__(256) k_pack_job_tiled(PackJob j, const float* __restrict__ w, bf16* __restrict__ hi, bf16* __restrict__ lo) {
  __shared__ float tile[PT][PT + 1][PTT];
  pack_job(tile, j, w, hi, lo);
}

template <int TC>
__device__ __forceinline__ void unpack_job_tiled(float (&tile)[PT][PT + 1][PTT], const PackJob& j, const float* __restrict__ g,
                                                 float* __restrict__ out) {
  const int T = TC ? TC : j.T;
  const bool tdst = j.mode == PACK_T_FLIPPED;   // ConvTranspose3d gradient layout [Ci][Co][T], taps flipped back
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

__device__ __forceinline__ void unpack_job(float (&tile)[PT][PT + 1][PTT], const PackJob& j, const float* g, float* out) {
  if (j.T == 27) unpack_job_tiled<27>(tile, j, g, out);
  else if (j.T == 1) unpack_job_tiled<1>(tile, j, g, out);
  else if (j.T == 8) unpack_job_tiled<8>(tile, j, g, out);
  else unpack_job_tiled<0>(tile, j, g, out);
}

__global__ void __launch_bounds__(256) k_unpack_all_tiled(PtrTable grads, const PackJob* __restrict__ jobs,
                                                         const uint8_t* __restrict__ ws) {
  __shared__ float tile[PT][PT + 1][PTT];
  const PackJob j = jobs[blockIdx.y];
  float* __restrict__ out = const_cast<float*>(reinterpret_cast<const float*>(grads.p[j.pidx]));
  const float* __restrict__ g = reinterpret_cast<const float*>(ws + j.off_hi);   // fp32 accumulator [T][Cip][Cop]
  unpack_job(tile, j, g, out);
}

// one tensor (the per-tensor C ABI entry points)
__global__ void __launch_bounds__(256) k_unpack_job_tiled(PackJob j, const float* __restrict__ g, float* __restrict__ out) {
  __shared__ float tile[PT][PT + 1][PTT];
  unpack_job(tile, j, g, out);
}

int launch_pack_all(const PtrTable& params, const PackJob* jobs_dev, int njobs, uint8_t* ws, bool split, cudaStream_t st) {
  if (njobs == 0) return OK;
  k_pack_all_tiled<<<dim3(256, njobs), 256, 0, st>>>(params, jobs_dev, ws, split ? 1 : 0);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

int launch_unpack_all(const PtrTable& grads, const PackJob* jobs_dev, int njobs, const uint8_t* ws, cudaStream_t st) {
  if (njobs == 0) return OK;
  k_unpack_all_tiled<<<dim3(256, njobs), 256, 0, st>>>(grads, jobs_dev, ws);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// The write phase of the pack stores 8-channel chunks of the padded extents; the tile holds up to 27 taps.
static int check_pack_shape(const char* what, int Cop, int Cip, int T) {
  B200_REQUIRE(Cop % 8 == 0 && Cip % 8 == 0 && Cop > 0 && Cip > 0, E_UNSUPPORTED,
               "%s: padded channel counts cop=%d, cip=%d must be positive multiples of 8", what, Cop, Cip);
  B200_REQUIRE(T >= 1 && T <= 27, E_UNSUPPORTED, "%s: taps=%d unsupported (1..27)", what, T);
  return OK;
}

int launch_pack_weights(const float* w, int Co, int Ci, int Cop, int Cip, int T, int mode, bf16* hi, bf16* lo, cudaStream_t st) {
  B200_TRY(check_pack_shape("pack_weights", Cop, Cip, T));
  B200_REQUIRE(mode >= PACK_FWD && mode <= PACK_T_FWD, E_INVALID, "pack_weights: mode=%d", mode);
  const PackJob j = {0, Co, Ci, Cop, Cip, T, mode, 0, 0};
  k_pack_job_tiled<<<256, 256, 0, st>>>(j, w, hi, lo);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

int launch_unpack_wgrad(const float* g, int Co, int Ci, int Cop, int Cip, int T, int mode, float* out, cudaStream_t st) {
  B200_TRY(check_pack_shape("unpack_wgrad", Cop, Cip, T));
  B200_REQUIRE(mode == PACK_FWD || mode == PACK_T_FLIPPED, E_INVALID, "unpack_wgrad: mode=%d (0 or 2)", mode);
  const PackJob j = {0, Co, Ci, Cop, Cip, T, mode, 0, 0};
  k_unpack_job_tiled<<<256, 256, 0, st>>>(j, g, out);
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
        load8(dy.lo, nullptr, v * dy.ld + cy * 8, gl);
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
          load8(a.lo, nullptr, v * a.ld + c * 8, xl);
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
