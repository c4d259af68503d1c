// Distance fields of the Hausdorff distance-transform loss (monai.losses.HausdorffDTLoss, Karimi & Salcudean 2019) on the
// device, without copying the prediction to the host for scipy.ndimage.distance_transform_edt.
//
// For each kept (n, c), V = N x C' of them, the prediction mask p > 0.5 (p = act(x) as the loss kernels form it) and the target
// mask t > 0.5 each get the field edt(mask) + edt(~mask): at every voxel the Euclidean distance, in voxels, to the nearest
// voxel of the other value.  A mask that is empty or full has the field 0.  Each mask takes two transforms (features: its
// foreground voxels, or its background voxels), and every voxel is a query of exactly one of them -- the one whose features
// have the other value.  Plane pl = (v * 2 + m) * 2 + k: mask m (0 prediction, 1 target), features of kind k (0 foreground,
// 1 background).
//
//   k_hd_rows     one block per row (n, d, h): the masks of every kept channel (softmax statistics from all C channels of the
//                 voxel, once), integer foreground counts, and along W the offset to the nearest feature of each kind
//   k_hd_cols_h   one thread per column (pl, d, w): lower envelope along H (edt.cuh)
//   k_hd_cols_d   one thread per column (v, h, w), all four planes of v in turn: the envelope along D evaluated at the query
//                 voxels, scipy's distance rounded to fp32, stored -- as the weight pdt^alpha + tdt^alpha of the loss, or as the
//                 two raw fields
//
// Nothing is read back to the host (the empty-or-full rule reads the device counts), no floating-point atomics.
#include "edt.cuh"

namespace b200 {
namespace {

using edt::kColThreads;
constexpr int kWords = B200_SURFACE_MAX_EXTENT / 32;

struct Geo {
  int N, C, Cp, lo, D, H, W;
  long long S, HW;
  int nwc;                                         // column chunks of kColThreads along W
};

struct Layout {
  size_t counts, dw, hw, total;
};

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// scratch, in order: foreground counts uint32 [V][2] (zeroed per call), W offsets int16 [V][2][2][S], (dh, dw) int16x2 [V][2][2][S]
int layout(int N, int Cp, int D, int H, int W, Layout* L) {
  B200_REQUIRE(N >= 1 && Cp >= 1 && D >= 1 && H >= 1 && W >= 1, E_INVALID,
               "hausdorff_dt: n, kept channels, d, h, w must be >= 1 (got %d, %d, %d, %d, %d)", N, Cp, D, H, W);
  B200_REQUIRE(D <= B200_SURFACE_MAX_EXTENT && H <= B200_SURFACE_MAX_EXTENT && W <= B200_SURFACE_MAX_EXTENT, E_UNSUPPORTED,
               "hausdorff_dt: extent %d x %d x %d; at most %d per axis", D, H, W, B200_SURFACE_MAX_EXTENT);
  B200_REQUIRE((long long)N * Cp <= B200_SURFACE_MAX_PAIRS, E_UNSUPPORTED, "hausdorff_dt: %d x %d (item, class) pairs; at most %d",
               N, Cp, B200_SURFACE_MAX_PAIRS);
  const size_t V = (size_t)N * Cp, S = (size_t)D * H * W;
  L->counts = align256(sizeof(uint32_t) * 2 * V);
  L->dw = align256(sizeof(int16_t) * 4 * V * S);
  L->hw = align256(sizeof(uint32_t) * 4 * V * S);
  L->total = L->counts + L->dw + L->hw;
  return OK;
}

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + __expf(-x)); }   // as the loss kernels (dice_ce.cu)

// grid (D * H, N), 32 * ceil(W / 32) threads: thread w of row (d, h) of sample n
template <int TK, int ACT>
__global__ void __launch_bounds__(B200_SURFACE_MAX_EXTENT) k_hd_rows(const float* __restrict__ x, const void* __restrict__ tgt, Geo g,
                                                                     int16_t* __restrict__ dw, uint32_t* __restrict__ counts) {
  __shared__ uint32_t bits[2][2][kWords];          // [mask][kind][word]
  const int n = blockIdx.y, d = blockIdx.x / g.H, h = blockIdx.x % g.H, w = threadIdx.x;
  const int nw = (g.W + 31) >> 5;
  const bool in = w < g.W;
  const long long s = ((long long)d * g.H + h) * g.W + w;
  const float* xn = x + (long long)n * g.C * g.S + s;
  // softmax over all C channels, as the loss kernels form it: max, then the sum of exponentials in channel order
  float m = -INFINITY, inv = 0.f;
  if (ACT == A_SOFTMAX && in) {
    for (int k = 0; k < g.C; ++k) m = fmaxf(m, __ldg(xn + k * g.S));
    float sum = 0.f;
    for (int k = 0; k < g.C; ++k) sum += __expf(__ldg(xn + k * g.S) - m);
    inv = 1.f / sum;
  }
  int lab = -1;
  if (TK < T_ONEHOT_U8 && in) {
    const long long l = TK == T_LABEL_U8 ? (long long)__ldg(static_cast<const uint8_t*>(tgt) + (long long)n * g.S + s)
                                         : __ldg(static_cast<const long long*>(tgt) + (long long)n * g.S + s);
    lab = (l >= 0 && l < g.C) ? (int)l : -1;
  }
  const unsigned valid = __ballot_sync(0xffffffffu, in);
  for (int c = g.lo; c < g.C; ++c) {
    bool pm = false, tm = false;
    if (in) {
      const float r = __ldg(xn + (long long)c * g.S);
      const float p = ACT == A_SOFTMAX ? __expf(r - m) * inv : ACT == A_SIGMOID ? sigm(r) : r;
      pm = p > 0.5f;
      const long long e = ((long long)n * g.C + c) * g.S + s;
      tm = TK == T_SOFT_F32    ? __ldg(static_cast<const float*>(tgt) + e) > 0.5f
           : TK == T_ONEHOT_U8 ? (float)__ldg(static_cast<const uint8_t*>(tgt) + e) > 0.5f
                               : lab == c;
    }
    const unsigned bp = __ballot_sync(0xffffffffu, pm), bt = __ballot_sync(0xffffffffu, tm);
    if ((threadIdx.x & 31) == 0) {
      const int i = threadIdx.x >> 5;
      bits[0][0][i] = bp; bits[0][1][i] = ~bp & valid;
      bits[1][0][i] = bt; bits[1][1][i] = ~bt & valid;
    }
    __syncthreads();
    const int v = n * g.Cp + c - g.lo;
    if (threadIdx.x < 2) {
      unsigned cnt = 0;
      for (int i = 0; i < nw; ++i) cnt += __popc(bits[threadIdx.x][0][i]);
      if (cnt) atomicAdd(counts + v * 2 + threadIdx.x, cnt);
    }
    if (in)
      for (int pk = 0; pk < 4; ++pk) dw[((long long)v * 4 + pk) * g.S + s] = edt::row_offset(bits[pk >> 1][pk & 1], nw, w);
    __syncthreads();
  }
}

// grid (D * nwc, 4 V)
__global__ void __launch_bounds__(kColThreads) k_hd_cols_h(Geo g, const int16_t* __restrict__ dw, uint32_t* __restrict__ hw) {
  __shared__ uint8_t stk_all[B200_SURFACE_MAX_EXTENT * kColThreads];
  const int d = blockIdx.x / g.nwc, w = (blockIdx.x % g.nwc) * kColThreads + threadIdx.x;
  if (w >= g.W) return;
  const long long off = (long long)blockIdx.y * g.S + (long long)d * g.HW + w;
  const edt::CostH F{dw + off, g.W, 1.0, 1.0};
  edt::cols_h(F, g.H, stk_all + threadIdx.x, hw + off);
}

// grid (H * nwc, V).  weight != nullptr: weight [V][S] = pdt^alpha + tdt^alpha; else pdt / tdt [V][S] (either may be nullptr)
__global__ void __launch_bounds__(kColThreads) k_hd_cols_d(Geo g, const int16_t* __restrict__ dw, const uint32_t* __restrict__ hw,
                                                           const uint32_t* __restrict__ counts, float alpha, float* __restrict__ weight,
                                                           float* __restrict__ pdt, float* __restrict__ tdt) {
  __shared__ uint8_t stk_all[B200_SURFACE_MAX_EXTENT * kColThreads];
  const int h = blockIdx.x / g.nwc, w = (blockIdx.x % g.nwc) * kColThreads + threadIdx.x;
  if (w >= g.W) return;
  const int v = blockIdx.y;
  const long long off = (long long)h * g.W + w;
  uint8_t* stk = stk_all + threadIdx.x;
  for (int m = 0; m < 2; ++m) {
    float* out = weight ? weight : (m ? tdt : pdt);
    if (!out) continue;
    out += (long long)v * g.S + off;
    const bool first = !weight || m == 0;          // the weight's prediction term is stored, its target term added
    const uint32_t cnt = counts[v * 2 + m];
    if (cnt == 0 || cnt == (uint32_t)g.S) {        // empty or full: the field is 0
      if (first)
        for (int x = 0; x < g.D; ++x) out[x * g.HW] = 0.f;
      continue;
    }
    for (int k = 0; k < 2; ++k) {
      const long long pl = ((long long)v * 2 + m) * 2 + k;
      const edt::CostD F{hw + pl * g.S + off, g.HW, 1.0, 1.0, 1.0};
      const int16_t* feat = dw + pl * g.S + off;   // W offset 0: a feature of this kind, else a query
      const int sites = edt::fh_envelope(F, g.D, stk);
      if (sites == 0) continue;                    // not reached: a mask that is neither empty nor full has both kinds
      edt::EnvelopeWalk<edt::CostD> walk(F, stk, sites, F.s2);
      for (int x = 0; x < g.D; ++x) {
        if (feat[x * g.HW] == 0) continue;
        const int i = walk.site(x);
        const float dist = edt::distance(i, x, F.col[i * F.step], 1.0, 1.0, 1.0);
        const float val = weight ? powf(dist, alpha) : dist;
        out[x * g.HW] = first ? val : out[x * g.HW] + val;
      }
    }
  }
}

// one channel: softmax and the label-map expansion do not apply (as the loss kernels read it)
int geometry(const DiceCEDesc& d, int N, int C, int D, int H, int W, Geo* g, int* kind, int* act) {
  B200_REQUIRE(N >= 1 && C >= 1, E_INVALID, "hausdorff_dt: n=%d c=%d", N, C);
  B200_REQUIRE(C <= 128, E_UNSUPPORTED, "hausdorff_dt: %d channels (at most 128)", C);
  B200_REQUIRE(d.act >= 0 && d.act <= 2, E_INVALID, "hausdorff_dt: act=%d (0 none, 1 sigmoid, 2 softmax)", d.act);
  B200_REQUIRE(d.target_kind >= 0 && d.target_kind <= 3, E_INVALID, "hausdorff_dt: target_kind=%d", d.target_kind);
  *kind = d.target_kind;
  *act = d.act;
  if (C == 1) {
    B200_REQUIRE(d.target_kind != T_LABEL_I64, E_UNSUPPORTED, "hausdorff_dt: one channel with an int64 target (pass uint8 or fp32)");
    if (*kind == T_LABEL_U8) *kind = T_ONEHOT_U8;
    if (*act == A_SOFTMAX) *act = A_NONE;
  }
  g->N = N; g->C = C;
  g->lo = (!d.include_background && C > 1) ? 1 : 0;
  g->Cp = C - g->lo;
  g->D = D; g->H = H; g->W = W;
  g->S = (long long)D * H * W; g->HW = (long long)H * W;
  g->nwc = ceil_div(W, kColThreads);
  Layout L;
  return layout(N, g->Cp, D, H, W, &L);
}

#define B200_HD_SWITCH(M)                                                        \
  switch (kind * 3 + act) {                                                      \
    case 0: M(0, 0); break; case 1: M(0, 1); break; case 2: M(0, 2); break;      \
    case 3: M(1, 0); break; case 4: M(1, 1); break; case 5: M(1, 2); break;      \
    case 6: M(2, 0); break; case 7: M(2, 1); break; case 8: M(2, 2); break;      \
    case 9: M(3, 0); break; case 10: M(3, 1); break; default: M(3, 2); break;    \
  }

}  // namespace

size_t hausdorff_dt_scratch_bytes(const DiceCEDesc& d, int N, int C, int D, int H, int W) {
  Geo g;
  int kind, act;
  if (geometry(d, N, C, D, H, W, &g, &kind, &act) != OK) return 0;
  Layout L;
  layout(N, g.Cp, D, H, W, &L);
  return L.total;
}

int launch_hausdorff_dt_fields(const DiceCEDesc& d, const float* logits, const void* target, int N, int C, int D, int H, int W,
                               float alpha, void* scratch, float* weight, float* pdt, float* tdt, cudaStream_t st) {
  B200_REQUIRE(logits && target && scratch, E_INVALID, "hausdorff_dt: null argument");
  B200_REQUIRE(weight || pdt || tdt, E_INVALID, "hausdorff_dt: no output requested");
  B200_REQUIRE(!weight || alpha > 0.f, E_UNSUPPORTED, "hausdorff_dt: alpha=%g (> 0)", (double)alpha);
  Geo g;
  int kind, act;
  B200_TRY(geometry(d, N, C, D, H, W, &g, &kind, &act));
  Layout L;
  layout(N, g.Cp, D, H, W, &L);
  const int V = N * g.Cp;
  char* base = static_cast<char*>(scratch);
  uint32_t* counts = reinterpret_cast<uint32_t*>(base);
  int16_t* dwb = reinterpret_cast<int16_t*>(base + L.counts);
  uint32_t* hwb = reinterpret_cast<uint32_t*>(base + L.counts + L.dw);
  B200_CHECK_CUDA(cudaMemsetAsync(counts, 0, L.counts, st));
  const int threads = 32 * ceil_div(W, 32);
#define B200_HD_ROWS(tk, ac) k_hd_rows<tk, ac><<<dim3(D * H, N), threads, 0, st>>>(logits, target, g, dwb, counts);
  B200_HD_SWITCH(B200_HD_ROWS)
#undef B200_HD_ROWS
  B200_CHECK_CUDA(cudaGetLastError());
  k_hd_cols_h<<<dim3(D * g.nwc, 4 * V), kColThreads, 0, st>>>(g, dwb, hwb);
  B200_CHECK_CUDA(cudaGetLastError());
  k_hd_cols_d<<<dim3(H * g.nwc, V), kColThreads, 0, st>>>(g, dwb, hwb, counts, alpha, weight, pdt, tdt);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

#undef B200_HD_SWITCH

}  // namespace b200
