// Exact separable Euclidean distance transform on the device (Felzenszwalb & Huttenlocher 2012), shared by the boundary-distance
// metrics (surface.cu) and the distance-weighted loss (hausdorff_dt.cu).
//
// A transform carries the offsets of the nearest feature voxel through its passes: along W from a ballot bitmask of the row,
// then the lower envelope of parabolas along H and along D.  Every envelope comparison is a cross-multiplication in fp64: with
// unit spacing all operands are integers below 2^53, so the nearest feature is exact, and the distance is
// sqrt(((dd s_d)^2 + (dh s_h)^2) + (dw s_w)^2) in fp64 rounded to fp32, as scipy.ndimage.distance_transform_edt forms it from
// its feature transform.
#pragma once
#include "kernels.h"

namespace b200 {
namespace edt {

constexpr int kColThreads = 128;                   // columns per block of the H and D passes
constexpr int16_t kNone = 0x7fff;                  // W pass: no feature voxel in the row
constexpr uint32_t kNone32 = 0x7fff7fffu;          // H pass: no feature voxel in the plane column

// W offset from w to the nearest set bit of bits[0..nw) (the row's features; the nearer of the two on a tie is the lower
// one), or kNone
__device__ __forceinline__ int16_t row_offset(const uint32_t* bits, int nw, int w) {
  const int i0 = w >> 5, b0 = w & 31;
  int left = -1, right = -1;
  for (int i = i0; i >= 0 && left < 0; --i) {          // nearest set bit at or below w
    const unsigned x = i == i0 ? bits[i] & (0xffffffffu >> (31 - b0)) : bits[i];
    if (x) left = i * 32 + 31 - __clz(x);
  }
  for (int i = i0; i < nw && right < 0; ++i) {         // nearest set bit at or above w
    const unsigned x = i == i0 ? bits[i] & (0xffffffffu << b0) : bits[i];
    if (x) right = i * 32 + __ffs(x) - 1;
  }
  int16_t off = kNone;
  if (left >= 0) off = (int16_t)(left - w);
  if (right >= 0 && (left < 0 || right - w < w - left)) off = (int16_t)(right - w);
  return off;
}

// Lower envelope of the parabolas F(i) + s2 (x - i)^2 - s2 x^2 over the sites with a finite cost, F(i) = cost(i) + s2 i^2.
// stk: this thread's stack of site indices (stride kColThreads).  Returns the number of envelope sites (0: no finite cost).
// sep(a, b) = (F(b) - F(a)) / (2 s2 (b - a)) is never divided out: both tests cross-multiply.
template <class Cost>
__device__ __forceinline__ int fh_envelope(const Cost& F, int n, uint8_t* stk) {
  int top = -1;
  double Fa = 0.0, Fb = 0.0;                     // F of stk[top - 1], stk[top]
  for (int q = 0; q < n; ++q) {
    const double Fq = F(q);
    if (!(Fq < INFINITY)) continue;
    while (top >= 1) {
      const int a = stk[(top - 1) * kColThreads], bb = stk[top * kColThreads];
      // pop b when sep(b, q) <= sep(a, b)
      if ((Fq - Fb) * (double)(bb - a) <= (Fb - Fa) * (double)(q - bb)) {
        --top;
        Fb = Fa;
        if (top >= 1) Fa = F(stk[(top - 1) * kColThreads]);
      } else {
        break;
      }
    }
    stk[++top * kColThreads] = (uint8_t)q;
    Fa = Fb;
    Fb = Fq;
  }
  return top + 1;
}

// walks the envelope for x = 0, 1, ...: the site nearest to x
template <class Cost>
struct EnvelopeWalk {
  const Cost& F;
  const uint8_t* stk;
  int sites, k;
  double s2, F0, F1;
  __device__ EnvelopeWalk(const Cost& f, const uint8_t* s, int n, double s2_) : F(f), stk(s), sites(n), k(0), s2(s2_) {
    F0 = F(stk[0]);
    F1 = sites > 1 ? F(stk[kColThreads]) : 0.0;
  }
  __device__ int site(int x) {
    // advance while sep(stk[k], stk[k + 1]) < x
    while (k + 1 < sites) {
      const int a = stk[k * kColThreads], b = stk[(k + 1) * kColThreads];
      if (!(F1 - F0 < 2.0 * s2 * (double)x * (double)(b - a))) break;
      ++k;
      F0 = F1;
      if (k + 1 < sites) F1 = F(stk[(k + 1) * kColThreads]);
    }
    return stk[k * kColThreads];
  }
};

struct CostH {   // F(h') = (dw s_w)^2 + s_h^2 h'^2 along one (d, w) column of the W offsets
  const int16_t* col;
  long long step;
  double sw, s2;
  __device__ double operator()(int i) const {
    const int16_t o = col[i * step];
    if (o == kNone) return INFINITY;
    const double a = o * sw;
    return a * a + s2 * (double)i * (double)i;
  }
};

// The H pass of one (d, w) column of n voxels: out[x * F.step] = (dh, dw) of the nearest feature of the plane (d, x), packed as
// int16 pairs, or kNone32
__device__ __forceinline__ void cols_h(const CostH& F, int n, uint8_t* stk, uint32_t* out) {
  const int sites = fh_envelope(F, n, stk);
  if (sites == 0) {
    for (int x = 0; x < n; ++x) out[(long long)x * F.step] = kNone32;
    return;
  }
  EnvelopeWalk<CostH> walk(F, stk, sites, F.s2);
  for (int x = 0; x < n; ++x) {
    const int i = walk.site(x);
    const int16_t o = F.col[i * F.step];
    out[(long long)x * F.step] = ((uint32_t)(uint16_t)(int16_t)(i - x) << 16) | (uint16_t)o;
  }
}

struct CostD {   // F(d') = (dh s_h)^2 + (dw s_w)^2 + s_d^2 d'^2 along one (h, w) column of the H pass
  const uint32_t* col;
  long long step;
  double sh, sw, s2;
  __device__ double operator()(int i) const {
    const uint32_t p = col[i * step];
    if (p == kNone32) return INFINITY;
    const double a = (int16_t)(p >> 16) * sh, b = (int16_t)(p & 0xffffu) * sw;
    return a * a + b * b + s2 * (double)i * (double)i;
  }
};

// the distance from voxel x of a D column to its nearest feature, site i of the D envelope with H-pass entry p: scipy's fp64
// expression rounded to fp32
__device__ __forceinline__ float distance(int i, int x, uint32_t p, double sd, double sh, double sw) {
  const double a = __dmul_rn((double)(i - x), sd), b = __dmul_rn((double)(int16_t)(p >> 16), sh),
               c = __dmul_rn((double)(int16_t)(p & 0xffffu), sw);
  return __double2float_rn(__dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)), __dmul_rn(c, c))));
}

}  // namespace edt
}  // namespace b200
