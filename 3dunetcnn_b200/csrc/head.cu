// The 1x1x1 head for 9..128 outputs on tensor cores (wgmma, bf16 operands from shared memory, fp32 accumulators).  At these widths the head
// is a GEMM with N = classes whose logits traffic outweighs any convolution layer; the SIMT head (elementwise.cu) keeps 1..8.
//
//   forward   logits[n][o][s] = act(sum_c x[v][c] w[o][c] + bias[o])           M = voxels, N = outputs, K = C
//   backward  dx[v][c] = sum_o g[v][o] w[o][c]                                 M = voxels, N = C, K = outputs
//             dw[o][c] = sum_v g[v][o] x[v][c],  dbias[o] = sum_v g[v][o]      M = outputs, N = C, K = voxels
//
// A CTA (two warpgroups) walks 128-voxel tiles (tile t, t + gridDim.x, ...), prefetching the next tile into registers while
// the tensor cores work on the current one from shared memory.  Tiles may straddle samples; voxels past the end read as zero.  Split precision
// (x.lo != nullptr) splits the fp32 weights and dlogits into bf16 hi + lo and issues three MMAs (hi*hi + hi*lo + lo*hi); bf16
// mode rounds them to bf16.  The backward CTA count depends on the shape alone and every CTA adds its tiles in a fixed order,
// so the weight and bias gradients (slot partials + k_sum_slots) are bit-reproducible.
#include "kernels.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kTile = 128;          // voxels per tile
constexpr int kThreads = 256;       // two warpgroups; warpgroup g owns voxel rows [64 g, 64 g + 64) of a tile
constexpr int kMaxC = 64;           // input channels (K of the forward, N of the backward GEMMs; padded to 64 with zeros)
constexpr int kBwdSlots = 132;      // backward CTAs at most = weight-gradient partial slots
constexpr int kES = kTile + 4;      // row pitch (fp32) of the forward epilogue tile [o][voxel]

// Every operand tile is [R rows][Kc cols] bf16 in the no-swizzle core-matrix layout: 8 rows x 16 bytes (8 columns) form one
// contiguous 128-byte core matrix, core matrices along the columns are adjacent (128 B apart) and 8-row groups are Kc / 8 * 128 B
// apart.  A tile is read as a K-major operand (rows = M / N, columns = K: cm_desc_k) or as an MN-major one (rows = K,
// columns = M / N: cm_desc_mn).  Without swizzle the two majors name the offsets the other way round: K-major takes LBO = the
// step between core matrices along K and SBO = the step between 8-row groups; MN-major takes SBO = the step between core
// matrices along M / N and LBO = the step between 8-row groups along K.  Tiles: x [voxel][c] (Kc = 64), w [o][c] (Kc = 64),
// dlogits [o][voxel] (Kc = 128).
__device__ __forceinline__ int cm_off(int r, int c, int kc) { return (r >> 3) * (kc * 8) + (c >> 3) * 64 + (r & 7) * 8 + (c & 7); }

__device__ __forceinline__ uint64_t cm_desc_k(const bf16* base, int r0, int c0, int kc) {
  return desc_from(desc_lo(smem_u32(base + cm_off(r0, c0, kc)), 128), desc_hi(kc * 16, GMMA_SW_NONE));
}
__device__ __forceinline__ uint64_t cm_desc_mn(const bf16* base, int r0, int c0, int kc) {
  return desc_from(desc_lo(smem_u32(base + cm_off(r0, c0, kc)), kc * 16), desc_hi(128, GMMA_SW_NONE));
}

// fp32 weights [n_out][C] -> bf16 hi (+ lo) [rows][64], zero outside n_out x C
__device__ __forceinline__ void stage_weights(const float* __restrict__ w, int n_out, int C, int rows, bool split, bf16* sW) {
  for (int i = threadIdx.x; i < rows * kMaxC; i += kThreads) {
    const int o = i / kMaxC, c = i - o * kMaxC;
    const float v = (o < n_out && c < C) ? w[o * C + c] : 0.f;
    const bf16 h = __float2bfloat16_rn(v);
    sW[cm_off(o, c, kMaxC)] = h;
    if (split) sW[rows * kMaxC + cm_off(o, c, kMaxC)] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}

// One tile of x in registers: 16-byte chunk k of this thread = voxel row (tid + 256 k) % 128, channels 8 * ((tid + 256 k) / 128);
// chunks past C or past the last voxel are zero, so the K padding of the shared tile is rewritten with zeros every tile.
struct XRegs { uint4 hi[4], lo[4]; };

__device__ __forceinline__ void load_x(const Act& x, long long v0, long long total, XRegs& r) {
  const int c8n = x.C / 8;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int i = threadIdx.x + kThreads * k;
    const int row = i & (kTile - 1), ch = i >> 7;
    const long long v = v0 + row;
    r.hi[k] = r.lo[k] = make_uint4(0, 0, 0, 0);
    if (ch < c8n && v < total) {
      r.hi[k] = *reinterpret_cast<const uint4*>(x.hi + v * x.ld + ch * 8);
      if (x.lo) r.lo[k] = *reinterpret_cast<const uint4*>(x.lo + v * x.ld + ch * 8);
    }
  }
}

__device__ __forceinline__ void store_x(const XRegs& r, bool split, bf16* sX) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int i = threadIdx.x + kThreads * k;
    const int off = cm_off(i & (kTile - 1), (i >> 7) * 8, kMaxC);
    *reinterpret_cast<uint4*>(sX + off) = r.hi[k];
    if (split) *reinterpret_cast<uint4*>(sX + kTile * kMaxC + off) = r.lo[k];
  }
}

template <int R>
__device__ __forceinline__ void zero(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) d[i] = 0.f;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ forward
// smem: weights [hi, lo][NP][64] | x tile [hi, lo][128][64], reused as the epilogue tile [NP][kES] fp32
// warpgroup g: D[64 voxels][NP] += x[64][16 k] * w^T[16 k][NP] as NP / 16 m64n16k16 MMAs per K step
template <int NT>
__global__ void __launch_bounds__(kThreads) k_head_mma(Act x, const float* __restrict__ w, const float* __restrict__ bias,
                                                       int n_out, int act_mode, float* __restrict__ logits) {
  constexpr int NP = 16 * NT;
  extern __shared__ __align__(128) uint8_t smem[];
  const int C = x.C, ksteps = (C + 15) / 16;
  const bool split = x.lo != nullptr;
  bf16* sW = reinterpret_cast<bf16*>(smem);
  bf16* sX = sW + 2 * NP * kMaxC;
  float* sE = reinterpret_cast<float*>(sX);
  const int wg = threadIdx.x >> 7, wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const long long S = (long long)x.D * x.H * x.W, total = x.voxels();
  const long long tiles = (total + kTile - 1) / kTile;

  stage_weights(w, n_out, C, NP, split, sW);
  XRegs xr;
  if (blockIdx.x < tiles) load_x(x, (long long)blockIdx.x * kTile, total, xr);

  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    __syncthreads();   // the previous epilogue has read sE (which overlays sX)
    store_x(xr, split, sX);
    fence_proxy_async();
    __syncthreads();
    if (tile + gridDim.x < tiles) load_x(x, (tile + gridDim.x) * kTile, total, xr);

    float acc[NT][8];
#pragma unroll
    for (int j = 0; j < NT; ++j) zero(acc[j]);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < kMaxC / 16; ++ks) {
      if (ks >= ksteps) break;
      const uint64_t ah = cm_desc_k(sX, 64 * wg, 16 * ks, kMaxC), al = cm_desc_k(sX + kTile * kMaxC, 64 * wg, 16 * ks, kMaxC);
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        const uint64_t bh = cm_desc_k(sW, 16 * j, 16 * ks, kMaxC);
        Wgmma<16>::mma<0, 0>(acc[j], ah, bh, 1);
        if (split) {
          Wgmma<16>::mma<0, 0>(acc[j], ah, cm_desc_k(sW + NP * kMaxC, 16 * j, 16 * ks, kMaxC), 1);
          Wgmma<16>::mma<0, 0>(acc[j], al, bh, 1);
        }
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < NT; ++j) wgmma_fence_regs(acc[j]);
    __syncthreads();   // every warpgroup is done with sX
    const int r0 = 64 * wg + 16 * wq + (lane >> 2);
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int o = 16 * j + 8 * i + 2 * (lane & 3);
        sE[o * kES + r0] = acc[j][4 * i];
        sE[(o + 1) * kES + r0] = acc[j][4 * i + 1];
        sE[o * kES + r0 + 8] = acc[j][4 * i + 2];
        sE[(o + 1) * kES + r0 + 8] = acc[j][4 * i + 3];
      }
    __syncthreads();

    // epilogue: thread <-> voxel i of the tile; the two halves of the CTA take alternate channels, so a warp stores one
    // contiguous run of 32 voxels of one channel
    const int i = threadIdx.x & (kTile - 1), half = threadIdx.x >> 7;
    const long long v = tile * kTile + i;
    if (act_mode == 2 && half == 0 && v < total) {   // softmax over the n_out real channels of the voxel
      float m = -INFINITY;
      for (int o = 0; o < n_out; ++o) {
        float r = sE[o * kES + i];
        if (bias) r += __ldg(bias + o);
        sE[o * kES + i] = r;
        m = fmaxf(m, r);
      }
      float z = 0.f;
      for (int o = 0; o < n_out; ++o) { const float e = __expf(sE[o * kES + i] - m); sE[o * kES + i] = e; z += e; }
      for (int o = 0; o < n_out; ++o) sE[o * kES + i] /= z;
    }
    if (act_mode == 2) __syncthreads();
    if (v < total) {
      const long long n = v / S, s = v - n * S;
      float* out = logits + n * n_out * S + s;
      for (int o = half; o < n_out; o += 2) {
        float r = sE[o * kES + i];
        if (act_mode != 2 && bias) r += __ldg(bias + o);
        if (act_mode == 1) r = 1.f / (1.f + __expf(-r));
        out[(long long)o * S] = r;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward
// smem: weights [hi, lo][NP][64] | x tile [hi, lo][128][64] | dlogits tile [hi, lo][NG][128] (NG = NP rounded up to 64) |
// bias-gradient reduction [8 warps][NP] fp32
//   dx (warpgroup g: 64 voxels x 64 channels, K = NP outputs): A = dlogits tile read MN-major, B = weights read MN-major
//   dw (warpgroup g: outputs [64 g, 64 g + 64) x 64 channels, K = 128 voxels): A = dlogits K-major, B = x tile MN-major
// part: [gridDim.x][n_out][C] weight-gradient slots, then (dbias) [gridDim.x][n_out] bias-gradient slots
template <int NT>
__global__ void __launch_bounds__(kThreads, 1) k_head_bwd_mma(Act x, const float* __restrict__ w, int n_out,
                                                              const float* __restrict__ dlogits, Act dx, int want_dbias,
                                                              float* __restrict__ part) {
  constexpr int NP = 16 * NT;
  constexpr int NG = (NP + 63) / 64 * 64;
  constexpr int GV = 2 * NT;   // float4 of the dlogits tile per thread: NP rows x 32 float4 / 256 threads
  extern __shared__ __align__(128) uint8_t smem[];
  const int C = x.C, c8n = C / 8;
  const bool split = x.lo != nullptr;
  bf16* sW = reinterpret_cast<bf16*>(smem);
  bf16* sX = sW + 2 * NP * kMaxC;
  bf16* sG = sX + 2 * kTile * kMaxC;
  float* sB = reinterpret_cast<float*>(sG + 2 * NG * kTile);
  const int warp = threadIdx.x >> 5, wg = threadIdx.x >> 7, wq = warp & 3, lane = threadIdx.x & 31;
  const long long S = (long long)x.D * x.H * x.W, total = x.voxels();
  const long long tiles = (total + kTile - 1) / kTile;
  // float4 loads need S % 4 == 0 (a voxel quad 4 q.. of a tile then stays in one sample) and a 16-byte aligned dlogits: a
  // contiguous torch gradient may sit at any float offset of its storage
  const bool vec = (S & 3) == 0 && (reinterpret_cast<uintptr_t>(dlogits) & 15) == 0;
  // float4 k of this thread: output o = 8 k + tid % 8, voxels 4 q .. 4 q + 3 of the tile with q = tid / 8 (four lanes read 64
  // contiguous bytes of one output; eight outputs share one 128-byte core-matrix column block in shared memory)
  const int oq = threadIdx.x & 7, q = threadIdx.x >> 3;

  stage_weights(w, n_out, C, NP, split, sW);
  for (int i = threadIdx.x; i < 2 * NG * kTile; i += kThreads) sG[i] = __float2bfloat16_rn(0.f);   // rows NP..NG stay zero

  auto load_g = [&](long long v0, float4 (&r)[GV]) {
#pragma unroll
    for (int k = 0; k < GV; ++k) {
      const int o = 8 * k + oq;
      const long long v = v0 + 4 * q;
      r[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (o < n_out && v < total) {
        if (vec) {   // 4 voxels of one sample at a multiple of 4 floats from the aligned base
          const long long n = v / S;
          r[k] = __ldg(reinterpret_cast<const float4*>(dlogits + (n * n_out + o) * S + (v - n * S)));
        } else {   // S % 4 != 0 or a misaligned dlogits: the same float4, one voxel at a time
          float e[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const long long u = v + j, n = u / S;
            e[j] = u < total ? __ldg(dlogits + (n * n_out + o) * S + (u - n * S)) : 0.f;
          }
          r[k] = make_float4(e[0], e[1], e[2], e[3]);
        }
      }
    }
  };

  float dw[32], db[GV];
  zero(dw);
#pragma unroll
  for (int k = 0; k < GV; ++k) db[k] = 0.f;

  XRegs xr;
  float4 gr[GV];
  if (blockIdx.x < tiles) {
    load_x(x, (long long)blockIdx.x * kTile, total, xr);
    load_g((long long)blockIdx.x * kTile, gr);
  }

  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    __syncthreads();   // the previous tile's MMAs have completed (wgmma_wait) in every warpgroup
    store_x(xr, split, sX);
#pragma unroll
    for (int k = 0; k < GV; ++k) {
      const float e[4] = {gr[k].x, gr[k].y, gr[k].z, gr[k].w};
      db[k] += (e[0] + e[1]) + (e[2] + e[3]);
      uint32_t h[2], l[2];
      h[0] = pack_bf16x2(e[0], e[1]);
      h[1] = pack_bf16x2(e[2], e[3]);
      l[0] = pack_bf16x2(e[0] - bf16_lo_to_f(h[0]), e[1] - bf16_hi_to_f(h[0]));
      l[1] = pack_bf16x2(e[2] - bf16_lo_to_f(h[1]), e[3] - bf16_hi_to_f(h[1]));
      const int off = cm_off(8 * k + oq, 4 * q, kTile);
      *reinterpret_cast<uint2*>(sG + off) = make_uint2(h[0], h[1]);
      if (split) *reinterpret_cast<uint2*>(sG + NG * kTile + off) = make_uint2(l[0], l[1]);
    }
    fence_proxy_async();
    __syncthreads();
    if (tile + gridDim.x < tiles) {
      load_x(x, (tile + gridDim.x) * kTile, total, xr);
      load_g((tile + gridDim.x) * kTile, gr);
    }

    float acc[32];
    zero(acc);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < NT; ++ks) {   // dx = g w
      const uint64_t ah = cm_desc_mn(sG, 16 * ks, 64 * wg, kTile), bh = cm_desc_mn(sW, 16 * ks, 0, kMaxC);
      Wgmma<64>::mma<1, 1>(acc, ah, bh, 1);
      if (split) {
        Wgmma<64>::mma<1, 1>(acc, ah, cm_desc_mn(sW + NP * kMaxC, 16 * ks, 0, kMaxC), 1);
        Wgmma<64>::mma<1, 1>(acc, cm_desc_mn(sG + NG * kTile, 16 * ks, 64 * wg, kTile), bh, 1);
      }
    }
    if (64 * wg < NP) {
#pragma unroll
      for (int ks = 0; ks < kTile / 16; ++ks) {   // dw += g^T x
        const uint64_t ah = cm_desc_k(sG, 64 * wg, 16 * ks, kTile), bh = cm_desc_mn(sX, 16 * ks, 0, kMaxC);
        Wgmma<64>::mma<0, 1>(dw, ah, bh, 1);
        if (split) {
          Wgmma<64>::mma<0, 1>(dw, ah, cm_desc_mn(sX + kTile * kMaxC, 16 * ks, 0, kMaxC), 1);
          Wgmma<64>::mma<0, 1>(dw, cm_desc_k(sG + NG * kTile, 64 * wg, 16 * ks, kTile), bh, 1);
        }
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    wgmma_fence_regs(dw);

    const long long va = tile * kTile + 64 * wg + 16 * wq + (lane >> 2), vb = va + 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (j < c8n) {
        const int c = j * 8 + 2 * (lane & 3);
        const uint32_t ha = pack_bf16x2(acc[4 * j], acc[4 * j + 1]), hb = pack_bf16x2(acc[4 * j + 2], acc[4 * j + 3]);
        if (va < total) {
          *reinterpret_cast<uint32_t*>(dx.hi + va * dx.ld + c) = ha;
          if (dx.lo)
            *reinterpret_cast<uint32_t*>(dx.lo + va * dx.ld + c) =
                pack_bf16x2(acc[4 * j] - bf16_lo_to_f(ha), acc[4 * j + 1] - bf16_hi_to_f(ha));
        }
        if (vb < total) {
          *reinterpret_cast<uint32_t*>(dx.hi + vb * dx.ld + c) = hb;
          if (dx.lo)
            *reinterpret_cast<uint32_t*>(dx.lo + vb * dx.ld + c) =
                pack_bf16x2(acc[4 * j + 2] - bf16_lo_to_f(hb), acc[4 * j + 3] - bf16_hi_to_f(hb));
        }
      }
    }
  }

  // this CTA's slot of the partial sums
  const int nc = n_out * C;
  float* pw = part + (long long)blockIdx.x * nc;
  if (64 * wg < NP) {
    const int o = 64 * wg + 16 * wq + (lane >> 2);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = j * 8 + 2 * (lane & 3);
      if (j < c8n) {
        if (o < n_out) { pw[o * C + c] = dw[4 * j]; pw[o * C + c + 1] = dw[4 * j + 1]; }
        if (o + 8 < n_out) { pw[(o + 8) * C + c] = dw[4 * j + 2]; pw[(o + 8) * C + c + 1] = dw[4 * j + 3]; }
      }
    }
  }
  if (want_dbias) {   // lanes l, l ^ 8, l ^ 16, l ^ 24 share an output; then the 8 warps in order
#pragma unroll
    for (int k = 0; k < GV; ++k) {
      float s = db[k];
      s += __shfl_xor_sync(0xffffffffu, s, 8);
      s += __shfl_xor_sync(0xffffffffu, s, 16);
      if (lane < 8) sB[warp * NP + 8 * k + lane] = s;
    }
    __syncthreads();
    float* pb = part + (long long)gridDim.x * nc + (long long)blockIdx.x * n_out;
    for (int o = threadIdx.x; o < n_out; o += kThreads) {
      float s = 0.f;
      for (int i = 0; i < kThreads / 32; ++i) s += sB[i * NP + o];
      pb[o] = s;
    }
  }
}

// ------------------------------------------------------------------------------------------------ launchers
static size_t fwd_smem(int NP) {
  const size_t xtile = 2 * kTile * kMaxC * sizeof(bf16), etile = (size_t)NP * kES * sizeof(float);
  return 2 * NP * kMaxC * sizeof(bf16) + (xtile > etile ? xtile : etile);
}
static size_t bwd_smem(int NP) {
  const size_t NG = (NP + 63) / 64 * 64;
  return (2 * NP * kMaxC + 2 * kTile * kMaxC + 2 * NG * kTile) * sizeof(bf16) + (kThreads / 32) * NP * sizeof(float);
}

static long long head_tiles(const Act& x) { return (x.voxels() + kTile - 1) / kTile; }

static int bwd_grid(const Act& x) {
  const long long t = head_tiles(x);
  return (int)(t < kBwdSlots ? (t > 0 ? t : 1) : kBwdSlots);
}

size_t head_mma_bwd_scratch_bytes(int n_out, int C) { return (size_t)kBwdSlots * ((size_t)n_out * C + n_out) * sizeof(float); }

template <int NT>
static int launch_fwd_nt(const Act& x, const float* w, const float* bias, int n_out, int act_mode, float* logits, cudaStream_t st) {
  B200_TRY(set_max_dynamic_smem<k_head_mma<NT>>((int)fwd_smem(16 * NT)));
  const long long t = head_tiles(x);
  const int grid = (int)(t < 2 * 132 ? (t > 0 ? t : 1) : 2 * 132);
  k_head_mma<NT><<<grid, kThreads, fwd_smem(16 * NT), st>>>(x, w, bias, n_out, act_mode, logits);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

template <int NT>
static int launch_bwd_nt(const Act& x, const float* w, int n_out, const float* dlogits, const Act& dx, int want_dbias, float* part,
                         cudaStream_t st) {
  B200_TRY(set_max_dynamic_smem<k_head_bwd_mma<NT>>((int)bwd_smem(16 * NT)));
  k_head_bwd_mma<NT><<<bwd_grid(x), kThreads, bwd_smem(16 * NT), st>>>(x, w, n_out, dlogits, dx, want_dbias, part);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

static int check_mma_shape(const Act& x, int n_out, const char* what) {
  B200_REQUIRE(n_out >= 1 && n_out <= B200_HEAD_MAX_OUTPUTS, E_UNSUPPORTED, "%s: n_outputs=%d unsupported (1..%d)", what, n_out,
               B200_HEAD_MAX_OUTPUTS);
  B200_REQUIRE(x.C % 8 == 0 && x.C <= kMaxC && x.ld % 8 == 0, E_UNSUPPORTED,
               "%s: %d input channels unsupported with more than 8 outputs (a multiple of 8, at most %d)", what, x.C, kMaxC);
  return OK;
}

#define B200_HEAD_NT_SWITCH(CALL)                                                                                    \
  switch ((n_out + 15) / 16) {                                                                                       \
    case 1: return CALL(1); case 2: return CALL(2); case 3: return CALL(3); case 4: return CALL(4);                  \
    case 5: return CALL(5); case 6: return CALL(6); case 7: return CALL(7); default: return CALL(8);                 \
  }

int launch_head_mma_fwd(const Act& x, const float* w, int n_out, int act_mode, float* logits, cudaStream_t st, const float* bias) {
  B200_TRY(check_mma_shape(x, n_out, "head"));
#define B200_FWD(nt) launch_fwd_nt<nt>(x, w, bias, n_out, act_mode, logits, st)
  B200_HEAD_NT_SWITCH(B200_FWD)
#undef B200_FWD
}

// part: head_mma_bwd_scratch_bytes(n_out, C); the caller reduces the slots (bwd_grid(x) of them) with k_sum_slots
int launch_head_mma_bwd(const Act& x, const float* w, int n_out, const float* dlogits, const Act& dx, int want_dbias, float* part,
                        int* slots, cudaStream_t st) {
  B200_TRY(check_mma_shape(x, n_out, "head_bwd"));
  B200_REQUIRE(dx.C == x.C && dx.ld % 8 == 0 && (dx.lo != nullptr) == (x.lo != nullptr), E_INVALID, "head_bwd: dx does not match x");
  *slots = bwd_grid(x);
#define B200_BWD(nt) launch_bwd_nt<nt>(x, w, n_out, dlogits, dx, want_dbias, part, st)
  B200_HEAD_NT_SWITCH(B200_BWD)
#undef B200_BWD
}

#undef B200_HEAD_NT_SWITCH

}  // namespace b200
