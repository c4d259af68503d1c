// Boundary-distance scores of binary segmentations on the device: Hausdorff distance (max or percentile), average surface
// distance and normalised surface Dice (MONAI HausdorffDistanceMetric, SurfaceDistanceMetric, SurfaceDiceMetric), without
// copying the masks to the host for scipy.ndimage.binary_erosion + distance_transform_edt.
//
// V = B x C' pairs (prediction, ground truth) of one D x H x W extent.  Direction k = 0 is pred -> gt (queries: the edge voxels
// of the prediction, features: the edge voxels of the ground truth), k = 1 the reverse.  Exact Euclidean distance transform,
// separable (Felzenszwalb & Huttenlocher 2012), carrying the offsets of the nearest feature through the passes:
//
//   k_sf_rows     one block per row (v, d, h): fg = (value == 1), edge = fg & ~erode6(fg) for both masks (outside = background),
//                 integer edge counts, and along W the offset to the nearest edge voxel of the row from a ballot bitmask
//   k_sf_cols_h   one thread per column (v, k, d, w): lower envelope of the parabolas (dw s_w)^2 + s_h^2 (h - h')^2 -> (dh, dw)
//   k_sf_cols_d   one thread per column (v, k, h, w): the same along D, evaluated only at the query voxels: the distance is
//                 sqrt(((dd s_d)^2 + (dh s_h)^2) + (dw s_w)^2) in fp64 rounded to fp32, as scipy's _morphology.py computes it
//                 from the feature transform and MONAI casts it.  Reduced in place: max (uint32 atomicMax of the bit pattern),
//                 count <= tau (integer atomics), fp64 sum per block (summed in block order by k_sf_finish); with a percentile
//                 the keys of each column are also stored compactly and counted into a 16-bit histogram
//   k_sf_rank     one block per (v, k): the two ranks floor / ceil of r = float(q) (n - 1), and the bin of each
//   k_sf_hist2    the low 16 bits of the keys in each rank's bin
//   k_sf_finish   one block per pair: the two order statistics, torch's lerp, and HD / ASD / NSD with MONAI's empty-mask rules
//
// Every envelope comparison is a cross-multiplication in fp64: with unit spacing all operands are integers below 2^53, so the
// nearest feature is exact and every distance equals scipy's bit for bit.  No floating-point atomics; nothing is read back.
#include "kernels.h"

namespace b200 {
namespace {

constexpr int kColThreads = 128;                   // columns per block of the H and D passes
constexpr int kBins = 1 << 16;                     // 16-bit digits of the two-pass select
constexpr int kSelThreads = 256;
constexpr int16_t kNone = 0x7fff;                  // W pass: no edge voxel in the row
constexpr uint32_t kNone32 = 0x7fff7fffu;          // H pass: no edge voxel in the plane column

struct Geo {
  int V, D, H, W, Cp;
  long long S, HW;
  int nwc;                                         // column chunks of kColThreads along W
  int dirs;                                        // 1: pred -> gt only, 2: both directions
};

struct Layout {
  size_t counts, hist1, hist2, sel, partial, dw, hw, keys, colcnt, total;
  int nblk;                                        // blocks of k_sf_cols_d per (v, k)
};

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// scratch, in order: [counters | hist1 | hist2] (zeroed per call; the histograms only with a percentile), select state, block
// partial sums, W offsets int16 [V][2][S], (dh, dw) int16x2 [V][2][S], keys uint32 [V][2][H*W][D], keys per column int32.
int layout(int V, int D, int H, int W, Layout* L) {
  B200_REQUIRE(V >= 1 && D >= 1 && H >= 1 && W >= 1, E_INVALID, "surface: pairs, d, h, w must be >= 1 (got %d, %d, %d, %d)", V, D, H,
               W);
  B200_REQUIRE(D <= B200_SURFACE_MAX_EXTENT && H <= B200_SURFACE_MAX_EXTENT && W <= B200_SURFACE_MAX_EXTENT, E_UNSUPPORTED,
               "surface: extent %d x %d x %d; at most %d per axis", D, H, W, B200_SURFACE_MAX_EXTENT);
  B200_REQUIRE(V <= B200_SURFACE_MAX_PAIRS, E_UNSUPPORTED, "surface: %d (item, class) pairs; at most %d per call", V,
               B200_SURFACE_MAX_PAIRS);
  const size_t P = 2 * (size_t)V, S = (size_t)D * H * W;
  L->nblk = H * ceil_div(W, kColThreads);
  L->counts = align256(sizeof(uint32_t) * 4 * P);  // edge counts [V][2], max bits [P], count <= tau [P]
  L->hist1 = align256(sizeof(uint32_t) * kBins * P);
  L->hist2 = align256(sizeof(uint32_t) * 2 * kBins * P);
  L->sel = align256(sizeof(uint32_t) * 4 * P);
  L->partial = align256(sizeof(double) * L->nblk * P);
  L->dw = align256(sizeof(int16_t) * P * S);
  L->hw = align256(sizeof(uint32_t) * P * S);
  L->keys = align256(sizeof(uint32_t) * P * S);
  L->colcnt = align256(sizeof(int32_t) * P * H * W);
  L->total = L->counts + L->hist1 + L->hist2 + L->sel + L->partial + L->dw + L->hw + L->keys + L->colcnt;
  return OK;
}

__device__ __forceinline__ bool fg_at(const SurfaceMask& m, long long base, int D, int H, int W, int d, int h, int w) {
  if (d < 0 || d >= D || h < 0 || h >= H || w < 0 || w >= W) return false;
  const long long e = base + d * m.stride[2] + h * m.stride[3] + w * m.stride[4];
  return m.dtype == 0 ? __ldg(static_cast<const uint8_t*>(m.data) + e) == 1 : __ldg(static_cast<const float*>(m.data) + e) == 1.0f;
}

__global__ void __launch_bounds__(B200_SURFACE_MAX_EXTENT) k_sf_rows(SurfaceMask pred, SurfaceMask gt, Geo g, int16_t* __restrict__ dw,
                                                                     uint32_t* __restrict__ ecount) {
  __shared__ uint32_t bits[2][B200_SURFACE_MAX_EXTENT / 32];
  const int v = blockIdx.y, d = blockIdx.x / g.H, h = blockIdx.x % g.H, w = threadIdx.x;
  const int b = v / g.Cp, c = v % g.Cp;
  const int nw = (g.W + 31) >> 5;
  for (int m = 0; m < 2; ++m) {
    const SurfaceMask& s = m ? gt : pred;
    const long long base = b * s.stride[0] + c * s.stride[1];
    bool e = false;
    if (w < g.W && fg_at(s, base, g.D, g.H, g.W, d, h, w)) {
      const bool interior = fg_at(s, base, g.D, g.H, g.W, d - 1, h, w) && fg_at(s, base, g.D, g.H, g.W, d + 1, h, w) &&
                            fg_at(s, base, g.D, g.H, g.W, d, h - 1, w) && fg_at(s, base, g.D, g.H, g.W, d, h + 1, w) &&
                            fg_at(s, base, g.D, g.H, g.W, d, h, w - 1) && fg_at(s, base, g.D, g.H, g.W, d, h, w + 1);
      e = !interior;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, e);
    if ((threadIdx.x & 31) == 0) bits[m][threadIdx.x >> 5] = bal;
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    unsigned n = 0;
    for (int i = 0; i < nw; ++i) n += __popc(bits[threadIdx.x][i]);
    if (n) atomicAdd(ecount + v * 2 + threadIdx.x, n);
  }
  if (w >= g.W) return;
  const int i0 = w >> 5, b0 = w & 31;
  for (int m = 0; m < 2; ++m) {
    int left = -1, right = -1;
    for (int i = i0; i >= 0 && left < 0; --i) {          // nearest set bit at or below w
      const unsigned x = i == i0 ? bits[m][i] & (0xffffffffu >> (31 - b0)) : bits[m][i];
      if (x) left = i * 32 + 31 - __clz(x);
    }
    for (int i = i0; i < nw && right < 0; ++i) {         // nearest set bit at or above w
      const unsigned x = i == i0 ? bits[m][i] & (0xffffffffu << b0) : bits[m][i];
      if (x) right = i * 32 + __ffs(x) - 1;
    }
    int16_t off = kNone;
    if (left >= 0) off = (int16_t)(left - w);
    if (right >= 0 && (left < 0 || right - w < w - left)) off = (int16_t)(right - w);
    dw[(long long)(v * 2 + m) * g.S + ((long long)d * g.H + h) * g.W + w] = off;
  }
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

__global__ void __launch_bounds__(kColThreads) k_sf_cols_h(Geo g, const int16_t* __restrict__ dw, const double* __restrict__ spacing,
                                                           uint32_t* __restrict__ hw) {
  __shared__ uint8_t stk_all[B200_SURFACE_MAX_EXTENT * kColThreads];
  const int d = blockIdx.x / g.nwc, w = (blockIdx.x % g.nwc) * kColThreads + threadIdx.x;
  if (w >= g.W) return;
  const int pl = blockIdx.y, v = pl / g.dirs, k = pl % g.dirs;
  const double* sp = spacing + (v / g.Cp) * 3;
  const long long off = (long long)d * g.HW + w;
  CostH F{dw + (long long)(v * 2 + 1 - k) * g.S + off, g.W, sp[2], sp[1] * sp[1]};
  uint8_t* stk = stk_all + threadIdx.x;
  uint32_t* out = hw + (long long)pl * g.S + off;
  const int sites = fh_envelope(F, g.H, stk);
  if (sites == 0) {
    for (int x = 0; x < g.H; ++x) out[(long long)x * g.W] = kNone32;
    return;
  }
  EnvelopeWalk<CostH> walk(F, stk, sites, F.s2);
  for (int x = 0; x < g.H; ++x) {
    const int i = walk.site(x);
    const int16_t o = F.col[i * F.step];
    out[(long long)x * g.W] = ((uint32_t)(uint16_t)(int16_t)(i - x) << 16) | (uint16_t)o;
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

__global__ void __launch_bounds__(kColThreads) k_sf_cols_d(Geo g, const int16_t* __restrict__ dw, const uint32_t* __restrict__ hw,
                                                           const double* __restrict__ spacing, const float* __restrict__ tau, int select,
                                                           uint32_t* __restrict__ maxbits, uint32_t* __restrict__ nle,
                                                           double* __restrict__ partial, uint32_t* __restrict__ keys,
                                                           int32_t* __restrict__ colcnt, uint32_t* __restrict__ hist1) {
  __shared__ uint8_t stk_all[B200_SURFACE_MAX_EXTENT * kColThreads];
  __shared__ double wsum[kColThreads / 32];
  __shared__ float wmax[kColThreads / 32];
  __shared__ unsigned wcnt[kColThreads / 32];
  const int h = blockIdx.x / g.nwc, w = (blockIdx.x % g.nwc) * kColThreads + threadIdx.x;
  const int pl = blockIdx.y, v = pl / g.dirs, k = pl % g.dirs;
  const double* sp = spacing + (v / g.Cp) * 3;
  const float t = tau ? tau[v % g.Cp] : -1.f;
  float mx = 0.f;
  double sum = 0.0;
  unsigned cnt = 0;
  if (w < g.W) {
    const long long off = (long long)h * g.W + w;
    CostD F{hw + (long long)pl * g.S + off, g.HW, sp[1], sp[2], sp[0] * sp[0]};
    const int16_t* query = dw + (long long)(v * 2 + k) * g.S + off;   // W offset 0 = an edge voxel of the query mask
    uint8_t* stk = stk_all + threadIdx.x;
    const int sites = fh_envelope(F, g.D, stk);
    int nk = 0;
    if (sites > 0) {
      uint32_t* kc = keys + ((long long)pl * g.HW + off) * g.D;
      uint32_t* h1 = hist1 + (long long)pl * kBins;
      EnvelopeWalk<CostD> walk(F, stk, sites, F.s2);
      for (int x = 0; x < g.D; ++x) {
        if (query[x * g.HW] != 0) continue;
        const int i = walk.site(x);
        const uint32_t p = F.col[i * F.step];
        const double a = __dmul_rn((double)(i - x), sp[0]), b = __dmul_rn((double)(int16_t)(p >> 16), sp[1]),
                     c = __dmul_rn((double)(int16_t)(p & 0xffffu), sp[2]);
        const float dist = __double2float_rn(__dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)), __dmul_rn(c, c))));
        mx = fmaxf(mx, dist);
        sum += (double)dist;
        cnt += dist <= t;
        if (select) {
          const uint32_t key = __float_as_uint(dist);
          kc[nk++] = key;
          atomicAdd(h1 + (key >> 16), 1u);
        }
      }
    }
    if (select) colcnt[(long long)pl * g.HW + off] = nk;
  }
  // block reduction in a fixed order: the fp64 sum is the same every run
  for (int o = 16; o > 0; o >>= 1) {
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { wsum[wid] = sum; wmax[wid] = mx; wcnt[wid] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < kColThreads / 32; ++i) { sum += wsum[i]; mx = fmaxf(mx, wmax[i]); cnt += wcnt[i]; }
    partial[(long long)pl * gridDim.x + blockIdx.x] = sum;
    if (mx > 0.f) atomicMax(maxbits + pl, __float_as_uint(mx));   // non-negative floats order as their bit patterns
    if (cnt) atomicAdd(nle + pl, cnt);
  }
}

// The bin of the histogram h (kBins entries) holding 0-based rank r, and r within it: one block of kSelThreads.
__device__ void find_rank(const uint32_t* __restrict__ h, uint32_t r, uint32_t* bin, uint32_t* rem) {
  constexpr int kPer = kBins / kSelThreads;
  __shared__ uint32_t wsum[kSelThreads / 32];
  const uint32_t* own = h + threadIdx.x * kPer;
  uint32_t s = 0;
  for (int j = 0; j < kPer; ++j) s += own[j];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t inc = s;
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) wsum[wid] = inc;
  __syncthreads();
  uint32_t before = inc - s;
  for (int i = 0; i < wid; ++i) before += wsum[i];
  if (s > 0 && before <= r && r - before < s) {
    uint32_t q = r - before;
    for (int j = 0; j < kPer; ++j) {
      if (q < own[j]) { *bin = threadIdx.x * kPer + j; *rem = q; break; }
      q -= own[j];
    }
  }
  __syncthreads();
}

struct Ranks {
  uint32_t lo, hi;
  float w;
};

// torch.quantile on fp32: r = float(q) * (n - 1) in fp32, the order statistics at floor(r) and ceil(r), weight r - floor(r)
__device__ __forceinline__ Ranks ranks_of(float q, uint32_t n) {
  const float r = __fmul_rn(q, (float)(n - 1));
  Ranks R;
  R.lo = (uint32_t)floorf(r);
  R.hi = (uint32_t)ceilf(r);
  R.w = __fsub_rn(r, (float)R.lo);
  return R;
}

// sel[pl] = (bin of lo, rank in it, bin of hi, rank in it); 0xffffffff in the first word: nothing to select
__global__ void __launch_bounds__(kSelThreads) k_sf_rank(Geo g, float q, const uint32_t* __restrict__ ecount,
                                                         const uint32_t* __restrict__ hist1, uint32_t* __restrict__ sel) {
  __shared__ uint32_t res[4];
  const int pl = blockIdx.x, v = pl / g.dirs, k = pl % g.dirs;
  const uint32_t n = ecount[v * 2 + k], nf = ecount[v * 2 + 1 - k];
  if (n == 0 || nf == 0) {
    if (threadIdx.x == 0) sel[pl * 4] = 0xffffffffu;
    return;
  }
  const Ranks R = ranks_of(q, n);
  const uint32_t* h = hist1 + (long long)pl * kBins;
  find_rank(h, R.lo, &res[0], &res[1]);
  find_rank(h, R.hi, &res[2], &res[3]);
  if (threadIdx.x < 4) sel[pl * 4 + threadIdx.x] = res[threadIdx.x];
}

__global__ void k_sf_hist2(Geo g, const uint32_t* __restrict__ sel, const uint32_t* __restrict__ keys,
                           const int32_t* __restrict__ colcnt, uint32_t* __restrict__ hist2) {
  const int pl = blockIdx.y;
  const long long col = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= g.HW || sel[pl * 4] == 0xffffffffu) return;
  const uint32_t b0 = sel[pl * 4], b1 = sel[pl * 4 + 2];
  const uint32_t* kc = keys + ((long long)pl * g.HW + col) * g.D;
  uint32_t* h = hist2 + (long long)pl * 2 * kBins;
  const int n = colcnt[(long long)pl * g.HW + col];
  for (int j = 0; j < n; ++j) {
    const uint32_t key = kc[j];
    if ((key >> 16) == b0) atomicAdd(h + (key & 0xffffu), 1u);
    if ((key >> 16) == b1) atomicAdd(h + kBins + (key & 0xffffu), 1u);
  }
}

// one block per pair: per direction the statistic (max or quantile), the fp64 sum of the block partials in block order, then
// the metrics.  hd_dirs / asd_dirs: 1 = pred -> gt only, 2 = both.
__global__ void __launch_bounds__(kSelThreads) k_sf_finish(Geo g, int nblk, float q, int hd_dirs, int asd_dirs,
                                                           const uint32_t* __restrict__ ecount, const uint32_t* __restrict__ maxbits,
                                                           const uint32_t* __restrict__ nle, const double* __restrict__ partial,
                                                           const uint32_t* __restrict__ sel, const uint32_t* __restrict__ hist2,
                                                           float* __restrict__ hd, float* __restrict__ asd, float* __restrict__ nsd) {
  __shared__ uint32_t res[2][2];
  const int v = blockIdx.x;
  const uint32_t n0 = ecount[v * 2], n1 = ecount[v * 2 + 1];
  const bool normal = n0 > 0 && n1 > 0;
  float stat[2] = {0.f, 0.f};
  double sum[2] = {0.0, 0.0};
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    if (k >= g.dirs || !normal) break;
    const int pl = v * g.dirs + k;
    if (q > 0.f) {
      const uint32_t* h = hist2 + (long long)pl * 2 * kBins;
      find_rank(h, sel[pl * 4 + 1], &res[0][0], &res[0][1]);
      find_rank(h + kBins, sel[pl * 4 + 3], &res[1][0], &res[1][1]);
      const float a = __uint_as_float(sel[pl * 4] << 16 | res[0][0]), b = __uint_as_float(sel[pl * 4 + 2] << 16 | res[1][0]);
      // torch.lerp as its vectorised CPU kernel evaluates it: fma(w, b - a, a), or fma(w - 1, b - a, b) for w >= 0.5
      const float w = ranks_of(q, k ? n1 : n0).w, dba = __fsub_rn(b, a);
      stat[k] = w < 0.5f ? __fmaf_rn(w, dba, a) : __fmaf_rn(__fsub_rn(w, 1.f), dba, b);
    } else {
      stat[k] = __uint_as_float(maxbits[pl]);
    }
    if (threadIdx.x == 0)
      for (int i = 0; i < nblk; ++i) sum[k] += partial[(long long)pl * nblk + i];
  }
  if (threadIdx.x != 0) return;
  const float nan = __int_as_float(0x7fffffff);
  const bool none = n0 == 0 && n1 == 0;
  if (hd) hd[v] = none ? nan : !normal ? INFINITY : hd_dirs == 2 ? fmaxf(stat[0], stat[1]) : stat[0];
  if (asd) {
    const double s = asd_dirs == 2 ? sum[0] + sum[1] : sum[0];
    const double n = asd_dirs == 2 ? (double)n0 + (double)n1 : (double)n0;
    asd[v] = none ? nan : !normal ? INFINITY : __double2float_rn(s / n);
  }
  if (nsd) {
    const float c = (float)(nle[v * 2] + nle[v * 2 + 1]), n = (float)(n0 + n1);
    nsd[v] = none ? nan : !normal ? 0.f : __fdiv_rn(c, n);
  }
}

}  // namespace

size_t surface_scratch_bytes(int nb, int nc, int d, int h, int w) {
  Layout L;
  if (nb < 1 || nc < 1 || (long long)nb * nc > B200_SURFACE_MAX_PAIRS) {
    set_error("surface: %d items x %d classes; 1..%d pairs per call", nb, nc, B200_SURFACE_MAX_PAIRS);
    return 0;
  }
  if (layout(nb * nc, d, h, w, &L) != OK) return 0;
  return L.total;
}

int launch_surface_distance(const SurfaceMask& pred, const SurfaceMask& gt, int nb, int nc, int d, int h, int w, const double* spacing,
                            float q, int hd_dirs, int asd_dirs, const float* tau, float* hd, float* asd, float* nsd, void* scratch,
                            cudaStream_t st) {
  B200_REQUIRE(pred.data && gt.data && spacing && scratch, E_INVALID, "surface: null argument");
  B200_REQUIRE(hd || asd || nsd, E_INVALID, "surface: no output requested");
  B200_REQUIRE(!nsd || tau, E_INVALID, "surface: surface Dice needs the class thresholds");
  B200_REQUIRE((pred.dtype == 0 || pred.dtype == 1) && (gt.dtype == 0 || gt.dtype == 1), E_INVALID,
               "surface: dtype must be 0 (bool / uint8) or 1 (fp32)");
  B200_REQUIRE(hd_dirs >= 1 && hd_dirs <= 2 && asd_dirs >= 1 && asd_dirs <= 2, E_INVALID, "surface: directions must be 1 or 2");
  B200_REQUIRE(q >= 0.f && q <= 1.f, E_INVALID, "surface: quantile %g outside [0, 1]", (double)q);
  B200_REQUIRE(surface_scratch_bytes(nb, nc, d, h, w) != 0, E_UNSUPPORTED, "%s", get_error());
  Layout L;
  layout(nb * nc, d, h, w, &L);
  Geo g;
  g.V = nb * nc; g.D = d; g.H = h; g.W = w; g.Cp = nc;
  g.S = (long long)d * h * w; g.HW = (long long)h * w;
  g.nwc = ceil_div(w, kColThreads);
  g.dirs = (hd && hd_dirs == 2) || (asd && asd_dirs == 2) || nsd ? 2 : 1;
  const bool select = hd && q > 0.f;
  const int P = g.V * g.dirs;

  char* base = static_cast<char*>(scratch);
  uint32_t* ecount = reinterpret_cast<uint32_t*>(base);
  uint32_t* maxbits = ecount + 2 * g.V;
  uint32_t* nle = maxbits + 2 * g.V;
  uint32_t* hist1 = reinterpret_cast<uint32_t*>(base + L.counts);
  uint32_t* hist2 = reinterpret_cast<uint32_t*>(base + L.counts + L.hist1);
  size_t o = L.counts + L.hist1 + L.hist2;
  uint32_t* sel = reinterpret_cast<uint32_t*>(base + o); o += L.sel;
  double* partial = reinterpret_cast<double*>(base + o); o += L.partial;
  int16_t* dwb = reinterpret_cast<int16_t*>(base + o); o += L.dw;
  uint32_t* hwb = reinterpret_cast<uint32_t*>(base + o); o += L.hw;
  uint32_t* keys = reinterpret_cast<uint32_t*>(base + o); o += L.keys;
  int32_t* colcnt = reinterpret_cast<int32_t*>(base + o);

  B200_CHECK_CUDA(cudaMemsetAsync(base, 0, select ? L.counts + L.hist1 + L.hist2 : L.counts, st));
  k_sf_rows<<<dim3(d * h, g.V), 32 * ceil_div(w, 32), 0, st>>>(pred, gt, g, dwb, ecount);
  B200_CHECK_CUDA(cudaGetLastError());
  k_sf_cols_h<<<dim3(d * g.nwc, P), kColThreads, 0, st>>>(g, dwb, spacing, hwb);
  B200_CHECK_CUDA(cudaGetLastError());
  k_sf_cols_d<<<dim3(h * g.nwc, P), kColThreads, 0, st>>>(g, dwb, hwb, spacing, nsd ? tau : nullptr, select, maxbits, nle, partial,
                                                          keys, colcnt, hist1);
  B200_CHECK_CUDA(cudaGetLastError());
  if (select) {
    k_sf_rank<<<P, kSelThreads, 0, st>>>(g, q, ecount, hist1, sel);
    B200_CHECK_CUDA(cudaGetLastError());
    k_sf_hist2<<<dim3(ceil_div(h * w, 256), P), 256, 0, st>>>(g, sel, keys, colcnt, hist2);
    B200_CHECK_CUDA(cudaGetLastError());
  }
  k_sf_finish<<<g.V, kSelThreads, 0, st>>>(g, L.nblk, select ? q : 0.f, hd_dirs, asd_dirs, ecount, maxbits, nle, partial, sel, hist2, hd,
                                           asd, nsd);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

}  // namespace b200
