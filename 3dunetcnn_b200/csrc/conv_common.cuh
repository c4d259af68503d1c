// Shared pieces of the implicit-GEMM convolution kernel (igemm_conv.cu): argument block, TMA map bundle and the fused
// epilogue.
#pragma once
#include "kernels.h"
#include "ptx.cuh"
#include "tmap.h"

namespace b200 {

struct ConvMaps {
  CUtensorMap a[2][2];  // [source][hi/lo]
  CUtensorMap b[2][2];
  CUtensorMap o[2];     // output tile stores (hi/lo): the epilogue stages 128 x BN tiles in shared memory and TMA-stores them
};
// parity-class mode of the streaming kernel (stride-2 data gradient): one output map per class and hi/lo
struct ConvClassMaps {
  CUtensorMap oc[8][2];
};

// Row `r` / 16-byte chunk `c` of a [128 rows][CB channels] bf16 staging tile laid out the way a TMA store with the
// matching 32B/64B/128B swizzle expects it (absolute-address XOR; the tile base is 1024-byte aligned).
template <int CB>
__device__ __forceinline__ uint32_t stage_off(int r, int c) {
  constexpr uint32_t RBO = CB * 2;
  constexpr uint32_t MASK = RBO >= 128 ? 7u : RBO >= 64 ? 3u : 1u;
  const uint32_t off = r * RBO + c * 16;
  return off ^ (((off >> 7) & MASK) << 4);
}

struct ConvArgs {
  int N, Do, Ho, Wo, Cout;
  int tw, th, td;
  int tiles_w, tiles_h, tiles_d;
  int ntaps[2], ksz[2], kchunks[2], stride[2], pad[2];
  int npass;
  int mode;
  int cls_pair;     // parity-class mode, single-pass bf16: the two W-parity classes share one 256-row staging tile and one dense store
  bf16* out_hi; bf16* out_lo; int ldo;
  const bf16* res_hi; const bf16* res_lo; int ldr;
  const float* scale;
  double* stats; int stats_ld;
  const bf16* x_hi; const bf16* x_lo; int ldx;
  const float4* coef; int coef_ld;
  float slope;
  double* bstats;
  const float* bias;   // optional per-output-channel bias (ConvTranspose3d, decoder.py:101-102)
  int zero_last;       // force the high boundary plane/row/column of the output to exactly 0 (F.pad after ConvT, unet.py:38)
  // parity-class mode (streaming kernel only; blockIdx.z = class (pd,ph,pw) = 4*pd + 2*ph + pw): the output tensor has
  // twice the source extent, class c computes out[2j + p] = sum over its tap list of src[j + delta] * W[tap].
  // cls_tap entry: bits 0-4 packed-weight tap index, bit 5 / 6 / 7 = delta_w / delta_h / delta_d (0 or +1).
  int cls_mode;
  unsigned char cls_n[8];
  unsigned char cls_tap[8][8];
};

// Transposing butterfly: every lane holds 16 column values of its own row; on return lane l holds the sum over the
// 32 rows of column ((l >> 1) & 15)  (lanes 2k and 2k+1 hold the same column).  16 shuffles instead of 80.
__device__ __forceinline__ float warp_colsum16(float (&v)[16], int lane) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const bool up = lane & 16;
    float send = up ? v[i] : v[i + 8];
    float keep = up ? v[i + 8] : v[i];
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const bool up = lane & 8;
    float send = up ? v[i] : v[i + 4];
    float keep = up ? v[i + 4] : v[i];
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const bool up = lane & 4;
    float send = up ? v[i] : v[i + 2];
    float keep = up ? v[i + 2] : v[i];
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  {
    const bool up = lane & 2;
    float send = up ? v[0] : v[1];
    float keep = up ? v[1] : v[0];
    v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  }
  return v[0] + __shfl_xor_sync(0xffffffffu, v[0], 1);
}


// L2 prefetch of the epilogue's side input (residual in mode 0, the norm's raw input in mode 1) for one output row.
// Issued at tile start, long before the accumulator is ready: the DRAM latency overlaps the MMAs, the later loads hit L2.
__device__ __forceinline__ void conv_epilogue_prefetch(const ConvArgs& p, int n0, int ncols, long long vox, bool valid) {
  const bf16* hi = p.mode == 0 ? p.res_hi : p.x_hi;
  if (!hi || !valid) return;
  const bf16* lo = p.mode == 0 ? p.res_lo : p.x_lo;
  const int ld = p.mode == 0 ? p.ldr : p.ldx;
  int c1 = n0 + ncols;
  if (c1 > p.Cout) c1 = p.Cout;
  for (int c = n0; c < c1; c += 64) {   // one 128-byte line per 64 channels
    asm volatile("prefetch.global.L2 [%0];" ::"l"(hi + vox * ld + c));
    if (lo) asm volatile("prefetch.global.L2 [%0];" ::"l"(lo + vox * ld + c));
  }
}

// Fused epilogue for one row of a 128-row fp32 accumulator tile in shared memory (`acc_row`: this thread's row).  Columns
// are processed in groups of <= 64: the group's side input (residual / norm input) is loaded into registers up front (one
// latency per group instead of one per 16-column chunk), then per 16-column chunk:
// accumulator -> (+residual)(*scale) | GN/ReLU backward -> hi/lo store -> per-channel partial sums into s_stats (slot `wslot`).
template <int BN>
__device__ __forceinline__ void conv_epilogue_tile(const ConvArgs& p, const float* acc_row, int wslot, int lane, int n,
                                                   int n0, long long vox, bool valid, float* s_stats,
                                                   const float4* s_coef, bool want_stats, bool edge, uint8_t* stage,
                                                   int row, bool split) {
  // `stage`: 1024-aligned shared staging tile [BN/CBO boxes][128 rows][CBO channels] (+ the lo tile OUT_TILE bytes
  // later in split mode); the caller TMA-stores it after a proxy fence + barrier.
  constexpr int G = BN < 64 ? BN : 64;
  constexpr int CBO = BN < 64 ? BN : 64;
  constexpr int OUT_BOX = 128 * CBO * 2;
  constexpr int OUT_TILE = 128 * BN * 2;
  const bf16* side_hi = p.mode == 0 ? p.res_hi : p.x_hi;
  const bf16* side_lo = p.mode == 0 ? p.res_lo : p.x_lo;
  const int side_ld = p.mode == 0 ? p.ldr : p.ldx;
#pragma unroll 1
  for (int g0 = 0; g0 < BN; g0 += G) {
    if (n0 + g0 >= p.Cout) break;
    uint4 ph[G / 8], pl[G / 8];
    if (side_hi && valid) {
#pragma unroll
      for (int i = 0; i < G / 8; ++i) {
        const int cc = n0 + g0 + i * 8;
        if (cc < p.Cout) {
          ph[i] = *reinterpret_cast<const uint4*>(side_hi + vox * side_ld + cc);
          if (side_lo) pl[i] = *reinterpret_cast<const uint4*>(side_lo + vox * side_ld + cc);
        }
      }
    }
#pragma unroll
    for (int jj = 0; jj < G / 16; ++jj) {
      const int j = g0 / 16 + jj;
      const int c0 = n0 + j * 16;
      if (c0 < p.Cout) {
        float v[16], q[16];
#pragma unroll
        for (int i = 0; i < 16; i += 4) {
          const float4 a = *reinterpret_cast<const float4*>(acc_row + j * 16 + i);
          v[i] = a.x; v[i + 1] = a.y; v[i + 2] = a.z; v[i + 3] = a.w;
        }
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const int cc = c0 + hf * 8;
          float* vv = v + hf * 8;
          float* qq = q + hf * 8;
          if (cc < p.Cout && valid) {
            float sv[8];
            if (side_hi) {
              const uint4 a = ph[jj * 2 + hf];
              sv[0] = bf16_lo_to_f(a.x); sv[1] = bf16_hi_to_f(a.x); sv[2] = bf16_lo_to_f(a.y); sv[3] = bf16_hi_to_f(a.y);
              sv[4] = bf16_lo_to_f(a.z); sv[5] = bf16_hi_to_f(a.z); sv[6] = bf16_lo_to_f(a.w); sv[7] = bf16_hi_to_f(a.w);
              if (side_lo) {
                const uint4 b = pl[jj * 2 + hf];
                sv[0] += bf16_lo_to_f(b.x); sv[1] += bf16_hi_to_f(b.x); sv[2] += bf16_lo_to_f(b.y); sv[3] += bf16_hi_to_f(b.y);
                sv[4] += bf16_lo_to_f(b.z); sv[5] += bf16_hi_to_f(b.z); sv[6] += bf16_lo_to_f(b.w); sv[7] += bf16_hi_to_f(b.w);
              }
            }
            if (p.mode == 0) {
              if (side_hi) {
#pragma unroll
                for (int i = 0; i < 8; ++i) vv[i] += sv[i];
              }
              if (p.scale) {
#pragma unroll
                for (int i = 0; i < 8; ++i) vv[i] *= __ldg(p.scale + (long long)n * p.Cout + cc + i);
              }
              if (p.bias) {
#pragma unroll
                for (int i = 0; i < 8; ++i) vv[i] += __ldg(p.bias + cc + i);
              }
              if (edge) {
#pragma unroll
                for (int i = 0; i < 8; ++i) vv[i] = 0.f;
              }
#pragma unroll
              for (int i = 0; i < 8; ++i) qq[i] = vv[i] * vv[i];
            } else {
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float4 k = s_coef[j * 16 + hf * 8 + i];
                const float z = fmaf(k.x, sv[i], k.y);
                const float dz = z > 0.f ? vv[i] : vv[i] * p.slope;
                vv[i] = dz;
                qq[i] = dz * (sv[i] - k.z) * k.w;
              }
            }
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) { vv[i] = 0.f; qq[i] = 0.f; }
          }
          {
            uint4 o;
            o.x = pack_bf16x2(vv[0], vv[1]); o.y = pack_bf16x2(vv[2], vv[3]);
            o.z = pack_bf16x2(vv[4], vv[5]); o.w = pack_bf16x2(vv[6], vv[7]);
            const int col = j * 16 + hf * 8;
            uint8_t* dst = stage + (col / CBO) * OUT_BOX + stage_off<CBO>(row, (col % CBO) / 8);
            *reinterpret_cast<uint4*>(dst) = o;
            if (split) {
              uint4 l;
              l.x = pack_bf16x2(vv[0] - bf16_lo_to_f(o.x), vv[1] - bf16_hi_to_f(o.x));
              l.y = pack_bf16x2(vv[2] - bf16_lo_to_f(o.y), vv[3] - bf16_hi_to_f(o.y));
              l.z = pack_bf16x2(vv[4] - bf16_lo_to_f(o.z), vv[5] - bf16_hi_to_f(o.z));
              l.w = pack_bf16x2(vv[6] - bf16_lo_to_f(o.w), vv[7] - bf16_hi_to_f(o.w));
              *reinterpret_cast<uint4*>(dst + OUT_TILE) = l;
            }
          }
        }
        if (want_stats) {
          const float s1 = warp_colsum16(v, lane);
          const float s2 = warp_colsum16(q, lane);
          if ((lane & 1) == 0) {
            // s_stats: one private [BN][2] slot per epilogue warp (no shared-memory float atomics: they are CAS loops)
            float2* mine = reinterpret_cast<float2*>(s_stats) + wslot * BN + j * 16 + ((lane >> 1) & 15);
            float2 acc = *mine;
            acc.x += s1; acc.y += s2;
            *mine = acc;
          }
        }
      }
    }
  }
}

}  // namespace b200
