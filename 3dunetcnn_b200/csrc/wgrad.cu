// Convolution weight gradient on the sm_90a tensor cores (wgmma).
//
//   dW[tap][ci][co] += sum_v  A[v*stride + tap - pad][ci] * dY[v][co]        (fp32 accumulate in registers)
//
// Replaces the bwd-filter half of nn.Conv3d autograd (reference unet3d/models/pytorch/classification/resnet.py:12-22 used
// by myronenko.py:15,20,43,104; backward driven by unet3d/train/training_utils.py:65-71).
// GEMM view (K = voxels, both operands "MN-major": the contraction index is the slow axis of NDHWC memory):
//   M side (128 rows)  = 128/CB (tap, ci-chunk) "units" of CB input channels each - every unit is one TMA box
//                        (CB, tw, th, td, 1) of the activation at that tap's shifted coordinate, placed LBO bytes
//                        apart so that a wgmma sees them as swizzle atoms along M.  For Cin = 32 four taps share one
//                        M tile, for Cin >= 128 one tap fills it - no padding waste for narrow layers.
//   N side (BN columns) = output channels of dY, one or two boxes of min(BN,64) channels.
//   K                   = the 128 voxels of a spatial tile, 8 steps of K=16 per tile, each two m64 wgmmas (the M halves).
// A CTA owns QT = 128/BN M-tiles (accumulators in the registers of its consumer warpgroup) and a contiguous range of voxel
// tiles (split-K); the dY tile of a voxel block is loaded once and reused by all of the CTA's M-tiles.  Partial sums are
// reduced into the fp32 gradient buffer with vector atomics.  Split-precision mode: passes (a_hi,dy_hi), (a_lo,dy_hi),
// (a_hi,dy_lo).
#include <algorithm>
#include <cstdlib>
#include "kernels.h"
#include "ptx.cuh"
#include "tmap.h"

namespace b200 {

struct WgradMaps {
  CUtensorMap a[2];   // hi / lo
  CUtensorMap dy[2];
};

struct WgradArgs {
  int N, Do, Ho, Wo;
  int Ci, Co, Cip, Cop;
  int tw, th, td, tiles_w, tiles_h, tiles_d;
  int ksz, stride, ntaps, pad;
  int nci;        // ci chunks per tap
  int units;      // ntaps * nci
  int qtiles;     // M-tiles in total
  int qt;         // M-tiles per CTA
  int kblocks;    // voxel tiles in total
  int splits;
  int npass;
  float* dw;
  float* part;             // deterministic mode: per-split partial sums [splits][T][Cip][Cop] (plain stores) instead of atomics
  long long part_stride;   // elements per split
};

constexpr int WG_A_STAGES = 4;
constexpr int WG_D_STAGES = 2;
constexpr int WG_A_BYTES = 32768;

// Halo mode (3x3x3 stride 1, 33..64 input channels, output planes filling an 8 x 16 tile, bf16): per voxel tile ONE TMA halo
// box (64, 10, 18, 3) of the activation replaces the 27 per-tap boxes; the A operand of tap (kd, kh, kw) is the box read from
// row kd * 180 + kh * 10 + kw with a K-group stride (SBO) of one 10-voxel halo row (the swizzle follows the absolute
// shared-memory address, as for the convolution's halo mode).  Two halo buffers: the producer loads the next tile's box while
// the MMAs of this one run.
constexpr int WG_HALO_TX = 540 * 128;
constexpr int WG_HALO_BYTES = (WG_HALO_TX + 1023) / 1024 * 1024;

template <int CB, int BN, bool HALO = false>
struct WgradCfg {
  static constexpr int CBN = BN < 64 ? BN : 64;
  static constexpr int BPM = 128 / CB;             // boxes per M tile
  static constexpr int BPN = BN / CBN;             // boxes per N tile
  static constexpr int QT = 128 / BN;              // M tiles per CTA: QT * BN fp32 accumulator registers per thread
  static constexpr int D_BYTES = BN * 128 * 2;
  static constexpr int D_STAGE = D_BYTES < 1024 ? 1024 : D_BYTES;
  static constexpr int A_REGION = HALO ? 2 * WG_HALO_BYTES : WG_A_STAGES * WG_A_BYTES;
  static constexpr int SMEM_BYTES = A_REGION + WG_D_STAGES * D_STAGE + 1024 + 1024;
  static_assert(!HALO || CB == 64, "halo mode reads 64-channel rows");
  static_assert(SMEM_BYTES <= 232448, "wgrad: configuration does not fit shared memory");
  static constexpr uint32_t LAYOUT_A = swizzle_for_row_bytes(CB * 2);
  static constexpr uint32_t LAYOUT_B = swizzle_for_row_bytes(CBN * 2);
  static constexpr uint32_t SBO_A = 16 * CB, LBO_A = 256 * CB;
  static constexpr uint32_t SBO_B = 16 * CBN, LBO_B = 256 * CBN;
  static constexpr uint32_t HALF_M = 64 / CB * LBO_A;   // bytes from M row 0 to M row 64
};

// Warps 0-3: one consumer warpgroup (wgmma issue and the write-back); warp 4: TMA producer.
template <int CB, int BN, bool HALO>
__global__ void __launch_bounds__(160, 1) k_wgrad(const __grid_constant__ WgradMaps maps, const WgradArgs p) {
  using Cfg = WgradCfg<CB, BN, HALO>;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment by pointer arithmetic on the __shared__ array: an integer round trip loses the address space and every
  // shared-memory access below would compile to a generic LD.E / ST.E instead of LDS / STS
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;
  uint8_t* smem_d = smem + Cfg::A_REGION;
  uint8_t* aux = smem_d + WG_D_STAGES * Cfg::D_STAGE;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(aux);
  uint64_t* a_empty = a_full + WG_A_STAGES;
  uint64_t* d_full = a_empty + WG_A_STAGES;
  uint64_t* d_empty = d_full + WG_D_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int split = blockIdx.x;
  const int q0 = blockIdx.y * p.qt;
  const int q1 = min(q0 + p.qt, p.qtiles);
  const int nq = q1 - q0;
  const int co0 = blockIdx.z * BN;
  const int kb0 = (int)((long long)p.kblocks * split / p.splits);
  const int kb1 = (int)((long long)p.kblocks * (split + 1) / p.splits);

  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&maps.a[0]);
    tma_prefetch_desc(&maps.dy[0]);
    for (int s = 0; s < WG_A_STAGES; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 4); }
    for (int s = 0; s < WG_D_STAGES; ++s) { mbar_init(&d_full[s], 1); mbar_init(&d_empty[s], 4); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();                 // set-up above overlaps the tail of the previous kernel; no global access before this line
  pdl_launch_dependents();
  const int pad = p.pad;

  if (warp == 4) {
    const uint32_t issue = elect_one() ? 1u : 0u;
    int ia = 0, id = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      int t = kb;
      const int wt = t % p.tiles_w; t /= p.tiles_w;
      const int ht = t % p.tiles_h; t /= p.tiles_h;
      const int dt = t % p.tiles_d;
      const int n = t / p.tiles_d;
      const int w0 = wt * p.tw, h0 = ht * p.th, d0 = dt * p.td;
      for (int pass = 0; pass < p.npass; ++pass) {
        {
          const int s = id % WG_D_STAGES;
          const uint32_t ph = (id / WG_D_STAGES) & 1;
          mbar_wait(&d_empty[s], ph ^ 1);
          mbar_expect_tx_if(issue, &d_full[s], Cfg::D_BYTES);
          uint8_t* dst = smem_d + s * Cfg::D_STAGE;
#pragma unroll
          for (int bx = 0; bx < Cfg::BPN; ++bx)
            tma_load_5d_if(issue, dst + bx * Cfg::LBO_B, &maps.dy[pass == 2], &d_full[s], co0 + bx * Cfg::CBN, w0, h0, d0, n);
          ++id;
        }
        if constexpr (HALO) {   // a_full / a_empty [0..1] guard the two halo buffers
          const int kbi = kb - kb0, hb = kbi & 1;
          mbar_wait(&a_empty[hb], ((kbi >> 1) & 1) ^ 1);
          mbar_expect_tx_if(issue, &a_full[hb], WG_HALO_TX);
          tma_load_5d_if(issue, smem_a + hb * WG_HALO_BYTES, &maps.a[0], &a_full[hb], 0, w0 - 1, h0 - 1, d0 - 1, n);
        } else {
        for (int q = q0; q < q1; ++q) {
          const int s = ia % WG_A_STAGES;
          const uint32_t ph = (ia / WG_A_STAGES) & 1;
          mbar_wait(&a_empty[s], ph ^ 1);
          mbar_expect_tx_if(issue, &a_full[s], WG_A_BYTES);
          uint8_t* dst = smem_a + s * WG_A_BYTES;
#pragma unroll
          for (int bx = 0; bx < Cfg::BPM; ++bx) {
            int u = q * Cfg::BPM + bx;
            if (u >= p.units) u = p.units - 1;  // duplicate a valid unit; its rows are never written back
            const int tap = u / p.nci, cic = u % p.nci;
            const int kd = tap / (p.ksz * p.ksz), kh = (tap / p.ksz) % p.ksz, kw = tap % p.ksz;
            tma_load_5d_if(issue, dst + bx * Cfg::LBO_A, &maps.a[pass == 1], &a_full[s], cic * CB,
                           w0 * p.stride + kw - pad, h0 * p.stride + kh - pad, d0 * p.stride + kd - pad, n);
          }
          ++ia;
        }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroup
  constexpr uint32_t hi_a = desc_hi(Cfg::SBO_A, Cfg::LAYOUT_A), hi_b = desc_hi(Cfg::SBO_B, Cfg::LAYOUT_B);
  const uint32_t a0 = smem_u32(smem_a), d0s = smem_u32(smem_d);
  float acc[Cfg::QT][2][BN / 2];
#pragma unroll
  for (int qi = 0; qi < Cfg::QT; ++qi)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { acc[qi][0][i] = 0.f; acc[qi][1][i] = 0.f; }
  int ia = 0, id = 0;
  int prev_a = -1, prev_d = -1;   // ring slots the previous wgmma group read: handed back once that group has retired
  for (int kb = kb0; kb < kb1; ++kb) {
    for (int pass = 0; pass < p.npass; ++pass) {
      const int sd = id % WG_D_STAGES;
      mbar_wait(&d_full[sd], (id / WG_D_STAGES) & 1);
      const uint32_t b_lo = desc_lo(d0s + sd * Cfg::D_STAGE, Cfg::LBO_B);
      if constexpr (HALO) {
        // M half hm of M tile q is unit 2q + hm = one tap of all 64 channels; K step k = output rows h = 2k, 2k + 1
        constexpr uint32_t hi_h = desc_hi(10 * 128, GMMA_SW128);
        const int kbi = kb - kb0, hb = kbi & 1;
        mbar_wait(&a_full[hb], (kbi >> 1) & 1);
        const uint32_t h_lo = desc_lo(a0 + hb * WG_HALO_BYTES, 16);
#pragma unroll
        for (int qi = 0; qi < Cfg::QT; ++qi) {
          if (qi < nq) {
            uint32_t off[2];
#pragma unroll
            for (int hm = 0; hm < 2; ++hm) {
              int u = (q0 + qi) * 2 + hm;
              if (u >= p.units) u = p.units - 1;   // duplicate a valid unit; its rows are never written back
              off[hm] = ((u / 9) * 180 + ((u / 3) % 3) * 10 + u % 3) * (128 >> 4);
            }
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              const uint64_t db = desc_from(b_lo + ((k * 2 * Cfg::SBO_B) >> 4), hi_b);
              Wgmma<BN>::template mma<1, 1>(acc[qi][0], desc_from(h_lo + off[0] + k * 20 * (128 >> 4), hi_h), db, 1u);
              Wgmma<BN>::template mma<1, 1>(acc[qi][1], desc_from(h_lo + off[1] + k * 20 * (128 >> 4), hi_h), db, 1u);
            }
            wgmma_commit();
          }
        }
        wgmma_wait<0>();   // this tile's box and dY stage are read: hand both back (the other halo buffer is already loading)
        if (lane == 0) {
          mbar_arrive(&d_empty[sd]);
          mbar_arrive(&a_empty[hb]);
        }
      } else {
#pragma unroll
      for (int qi = 0; qi < Cfg::QT; ++qi) {
        if (qi < nq) {
          const int sa = ia % WG_A_STAGES;
          mbar_wait(&a_full[sa], (ia / WG_A_STAGES) & 1);
          const uint32_t a_lo = desc_lo(a0 + sa * WG_A_BYTES, Cfg::LBO_A);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const uint64_t db = desc_from(b_lo + ((k * 2 * Cfg::SBO_B) >> 4), hi_b);
            Wgmma<BN>::template mma<1, 1>(acc[qi][0], desc_from(a_lo + ((k * 2 * Cfg::SBO_A) >> 4), hi_a), db, 1u);
            Wgmma<BN>::template mma<1, 1>(acc[qi][1], desc_from(a_lo + ((k * 2 * Cfg::SBO_A + Cfg::HALF_M) >> 4), hi_a), db, 1u);
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (lane == 0) {
            if (prev_a >= 0) mbar_arrive(&a_empty[prev_a]);
            if (prev_d >= 0) mbar_arrive(&d_empty[prev_d]);
          }
          prev_a = sa;
          prev_d = qi == nq - 1 ? sd : -1;
          ++ia;
        }
      }
      }
      ++id;
    }
  }
  wgmma_wait<0>();
#pragma unroll
  for (int qi = 0; qi < Cfg::QT; ++qi) { wgmma_fence_regs(acc[qi][0]); wgmma_fence_regs(acc[qi][1]); }
  if (lane == 0) {
    if (prev_a >= 0) mbar_arrive(&a_empty[prev_a]);
    if (prev_d >= 0) mbar_arrive(&d_empty[prev_d]);
  }

  // write-back straight from the fragments: element (row r, column c) -> dw[tap][ci][co0 + c]
  const bool has_work = kb1 > kb0;
  float* const base = p.part ? p.part + (long long)split * p.part_stride : p.dw;
#pragma unroll
  for (int qi = 0; qi < Cfg::QT; ++qi) {
    if (qi >= nq) continue;
#pragma unroll
    for (int hm = 0; hm < 2; ++hm) {
#pragma unroll
      for (int r8 = 0; r8 < 2; ++r8) {
        const int row = hm * 64 + warp * 16 + (lane >> 2) + r8 * 8;
        const int u = (q0 + qi) * Cfg::BPM + row / CB;
        const int tap = u / p.nci, cic = u % p.nci;
        const int ci = cic * CB + row % CB;
        if (u >= p.units || ci >= p.Ci || !(has_work || p.part)) continue;
        float* dst = base + ((long long)tap * p.Cip + ci) * p.Cop;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = co0 + j * 8 + 2 * (lane & 3);
          if (c < p.Cop) {   // Cop is a multiple of 4 and c is even: c + 1 < Cop as well
            const float2 v = make_float2(acc[qi][hm][4 * j + 2 * r8], acc[qi][hm][4 * j + 2 * r8 + 1]);
            if (p.part) *reinterpret_cast<float2*>(dst + c) = has_work ? v : make_float2(0.f, 0.f);   // every split writes its slot
            else atomicAdd(reinterpret_cast<float2*>(dst + c), v);
          }
        }
      }
    }
  }
}

static void pick_tile_w(int Wo, int Ho, int Do, int& tw, int& th, int& td) {
  tw = Wo >= 8 ? 8 : Wo >= 4 ? 4 : Wo >= 2 ? 2 : 1;
  int rem = 128 / tw;
  th = Ho >= 4 ? 4 : Ho >= 2 ? 2 : 1;
  if (th > rem) th = rem;
  td = rem / th;
}

template <int CB, int BN, bool HALO>
static int launch_wg(const WgradMaps& maps, const WgradArgs& a, dim3 grid, cudaStream_t st) {
  using Cfg = WgradCfg<CB, BN, HALO>;
  static bool attr_set[64] = {false};   // once per device: not a stream operation, keep it out of CUDA-graph captures
  int dev = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  if (dev >= 64 || !attr_set[dev]) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(k_wgrad<CB, BN, HALO>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    if (dev < 64) attr_set[dev] = true;
  }
  launch_pdl(k_wgrad<CB, BN, HALO>, grid, dim3(160), Cfg::SMEM_BYTES, st, maps, a);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// split-K factor of the streaming kernel for this shape (shared by the launcher and the deterministic-mode buffer sizing)
// halo mode (see WG_HALO_TX); B200UNET_NO_HALO=1 keeps every launch on per-tap boxes (A/B measurements)
static bool wgrad_halo_eligible(const WgradOp& op) {
  static const bool off = getenv("B200UNET_NO_HALO") && atoi(getenv("B200UNET_NO_HALO")) != 0;
  const Act& A = op.a;
  const Act& Y = op.dy;
  return !off && op.ksz == 3 && op.stride == 1 && !op.nopad && !A.lo && !Y.lo && A.C > 32 && A.C <= 64 && Y.W >= 8 && Y.H >= 16 &&
         A.D == Y.D && A.H == Y.H && A.W == Y.W;
}

static void wgrad_tile(bool halo, const WgradOp& op, int& tw, int& th, int& td) {
  if (halo) { tw = 8; th = 16; td = 1; }
  else pick_tile_w(op.dy.W, op.dy.H, op.dy.D, tw, th, td);
}

static int wgrad_stream_splits(const WgradOp& op, int num_sms, bool halo) {
  const Act& A = op.a;
  const Act& Y = op.dy;
  int tw, th, td;
  wgrad_tile(halo, op, tw, th, td);
  const int ntaps = op.ksz * op.ksz * op.ksz;
  const int CB = A.C > 32 ? 64 : A.C > 16 ? 32 : 16;
  const int BN = Y.C > 64 ? 128 : Y.C > 32 ? 64 : Y.C > 16 ? 32 : 16;
  const int qtiles = ceil_div(ntaps * ceil_div(A.C, CB), 128 / CB);
  int qt = 128 / BN;   // WgradCfg::QT
  if (qt > qtiles) qt = qtiles;
  const int groups = ceil_div(qtiles, qt);
  const int cotiles = ceil_div(Y.C, BN);
  const int kblocks = Y.N * ceil_div(Y.D, td) * ceil_div(Y.H, th) * ceil_div(Y.W, tw);
  int splits = num_sms / (groups * cotiles);
  if (splits < 1) splits = 1;
  if (splits > kblocks) splits = kblocks;
  return splits;
}

__global__ void k_wgrad_reduce(const float4* __restrict__ part, int splits, long long n4, float4* __restrict__ dw) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 acc = part[i];
    for (int s = 1; s < splits; ++s) {   // fixed order: bit-reproducible
      const float4 v = part[(long long)s * n4 + i];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    dw[i] = acc;
  }
}

int launch_wgrad_reduce(const float* part, int splits, long long elems, float* dw, cudaStream_t st) {
  B200_REQUIRE(part && dw && splits >= 1 && elems % 4 == 0, E_INVALID, "wgrad_reduce: bad argument");
  const long long n4 = elems / 4;
  long long blocks = (n4 + 255) / 256;
  if (blocks > 132 * 8) blocks = 132 * 8;
  k_wgrad_reduce<<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const float4*>(part), splits, n4, reinterpret_cast<float4*>(dw));
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

int device_sms() {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && sms > 0)
    return sms;
  cudaGetLastError();   // a host without a GPU (route queries, planning)
  return 132;
}

size_t wgrad_partial_bytes(const WgradOp& op, int num_sms) {
  const long long elems = (long long)op.ksz * op.ksz * op.ksz * op.Cip * op.Cop;
  // both tilings: a shape-only op (no lo pointers) cannot tell whether a split-precision launch will take halo mode
  const int splits = std::max(wgrad_stream_splits(op, num_sms, false), wgrad_halo_eligible(op) ? wgrad_stream_splits(op, num_sms, true) : 0);
  return (size_t)splits * elems * sizeof(float);
}

template <int CB_, int BN_, bool HALO_>
struct WgradKernel { static constexpr int CB = CB_, BN = BN_; static constexpr bool HALO = HALO_; };

// Every (CB, BN) of the per-tap kernel and every BN of the halo kernel (CB = 64) that the dispatch instantiates.
#define B200_WG_CONFIGS(X) \
  X(16, 16) X(16, 32) X(16, 64) X(16, 128) X(32, 16) X(32, 32) X(32, 64) X(32, 128) X(64, 16) X(64, 32) X(64, 64) X(64, 128)
#define B200_WG_HALO_CONFIGS(X) X(16) X(32) X(64) X(128)

// f(WgradKernel<CB, BN, HALO>{}) for the tensor-core kernel of route r: the one selection wgrad_route reports and launch_wgrad
// launches.  E_UNSUPPORTED when no such kernel is instantiated.
template <class F>
static int with_wgrad_kernel(const WgradRoute& r, F&& f) {
  if (r.kind == WGRAD_KIND_HALO) {
#define B200_WG_HALO_CASE(bn) \
    if (r.CB == 64 && r.BN == bn) return f(WgradKernel<64, bn, true>{});
    B200_WG_HALO_CONFIGS(B200_WG_HALO_CASE)
#undef B200_WG_HALO_CASE
  } else if (r.kind == WGRAD_KIND_TAP) {
#define B200_WG_CASE(cb, bn) \
    if (r.CB == cb && r.BN == bn) return f(WgradKernel<cb, bn, false>{});
    B200_WG_CONFIGS(B200_WG_CASE)
#undef B200_WG_CASE
  }
  set_error("wgrad: no kernel for CB=%d BN=%d (kind %d)", r.CB, r.BN, r.kind);
  return E_UNSUPPORTED;
}

int wgrad_route(const WgradOp& op, int num_sms, WgradRoute* r) {
  memset(r, 0, sizeof(*r));
  const Act& A = op.a;
  const Act& Y = op.dy;
  if (!op.part && wgrad_1x1_narrow_eligible(op)) {   // (the SIMT path reduces with atomics)
    B200_REQUIRE(A.N == Y.N && A.D == Y.D && A.H == Y.H && A.W == Y.W, E_INVALID, "wgrad_1x1_narrow: shape mismatch");
    r->kind = WGRAD_KIND_SIMT;
    r->ci8 = A.C / 8;
    r->npass = 1;
    return OK;
  }
  B200_REQUIRE(op.ksz == 1 || op.ksz == 3 || (op.ksz == 2 && op.nopad && op.stride == 2), E_UNSUPPORTED,
               "wgrad: kernel_size=%d unsupported", op.ksz);
  B200_REQUIRE(op.stride == 1 || op.stride == 2, E_UNSUPPORTED, "wgrad: stride=%d unsupported", op.stride);
  B200_REQUIRE(A.C % 8 == 0 && Y.C % 8 == 0 && A.ld % 8 == 0 && Y.ld % 8 == 0, E_UNSUPPORTED,
               "wgrad: channels must be multiples of 8 (Ci=%d Co=%d)", A.C, Y.C);
  B200_REQUIRE(op.Cop % 4 == 0 && op.Cop >= Y.C && op.Cip >= A.C, E_INVALID, "wgrad: bad accumulator pitch");
  const int pad = op.nopad ? 0 : op.ksz / 2;
  B200_REQUIRE((A.D + 2 * pad - op.ksz) / op.stride + 1 == Y.D && (A.H + 2 * pad - op.ksz) / op.stride + 1 == Y.H &&
                   (A.W + 2 * pad - op.ksz) / op.stride + 1 == Y.W && A.N == Y.N,
               E_INVALID, "wgrad: shape mismatch");
  const bool split = A.lo != nullptr || Y.lo != nullptr;
  if (split) B200_REQUIRE(A.lo && Y.lo, E_INVALID, "wgrad: split mode needs lo parts on both operands");
  const bool halo = wgrad_halo_eligible(op);
  r->kind = halo ? WGRAD_KIND_HALO : WGRAD_KIND_TAP;
  wgrad_tile(halo, op, r->tw, r->th, r->td);
  const int ntaps = op.ksz * op.ksz * op.ksz;
  r->CB = A.C > 32 ? 64 : A.C > 16 ? 32 : 16;
  r->BN = Y.C > 64 ? 128 : Y.C > 32 ? 64 : Y.C > 16 ? 32 : 16;
  r->nci = ceil_div(A.C, r->CB);
  r->units = ntaps * r->nci;
  r->qtiles = ceil_div(r->units, 128 / r->CB);
  r->QT = 128 / r->BN;   // WgradCfg::QT
  if (r->QT > r->qtiles) r->QT = r->qtiles;
  r->groups = ceil_div(r->qtiles, r->QT);
  r->QT = ceil_div(r->qtiles, r->groups);   // rebalance M tiles across groups
  r->cotiles = ceil_div(Y.C, r->BN);
  r->kblocks = Y.N * ceil_div(Y.D, r->td) * ceil_div(Y.H, r->th) * ceil_div(Y.W, r->tw);
  r->splits = wgrad_stream_splits(op, num_sms, halo);
  r->npass = split ? 3 : 1;
  r->part_bytes = (size_t)r->splits * ntaps * op.Cip * op.Cop * sizeof(float);
  return with_wgrad_kernel(*r, [](auto) { return (int)OK; });
}

int launch_wgrad(const WgradOp& op, cudaStream_t st) {
  WgradRoute r;
  B200_TRY(wgrad_route(op, device_sms(), &r));
  if (r.kind == WGRAD_KIND_SIMT) return launch_wgrad_1x1_narrow(op, st);
  const Act& A = op.a;
  const Act& Y = op.dy;
  B200_REQUIRE((reinterpret_cast<uintptr_t>(op.dw) & 15) == 0, E_INVALID, "wgrad: dw not 16B aligned");
  const bool split = r.npass == 3, halo = r.kind == WGRAD_KIND_HALO;

  WgradArgs a;
  memset(&a, 0, sizeof(a));
  WgradMaps maps;
  memset(&maps, 0, sizeof(maps));
  a.N = Y.N; a.Do = Y.D; a.Ho = Y.H; a.Wo = Y.W;
  a.Ci = A.C; a.Co = Y.C; a.Cip = op.Cip; a.Cop = op.Cop;
  a.tw = r.tw; a.th = r.th; a.td = r.td;
  a.tiles_w = ceil_div(Y.W, a.tw); a.tiles_h = ceil_div(Y.H, a.th); a.tiles_d = ceil_div(Y.D, a.td);
  a.ksz = op.ksz; a.stride = op.stride; a.ntaps = op.ksz * op.ksz * op.ksz; a.pad = op.nopad ? 0 : op.ksz / 2;
  const int CB = r.CB;
  const int CBN = r.BN < 64 ? r.BN : 64;
  a.nci = r.nci;
  a.units = r.units;
  a.qtiles = r.qtiles;
  a.qt = r.QT;
  a.kblocks = r.kblocks;
  a.splits = r.splits;
  a.npass = r.npass;
  a.dw = op.dw;
  if (op.part) {
    a.part = op.part;
    a.part_stride = (long long)a.ntaps * op.Cip * op.Cop;
    B200_REQUIRE(r.part_bytes <= op.part_bytes, E_INVALID, "wgrad: deterministic partial buffer too small (%d splits)", r.splits);
    if (op.part_splits) *op.part_splits = r.splits;
  }
  if (halo)   // one (64, 10, 18, 3) box around the 8 x 16 x 1 voxel tile; the zero padding is TMA out-of-bounds fill
    B200_TRY(make_act_map(&maps.a[0], A.hi, A.N, A.D, A.H, A.W, A.C, A.ld, 64, 10, 18, 3, 1, SWZ_128, A.vD, A.vH, A.vW));
  else
    B200_TRY(make_act_map(&maps.a[0], A.hi, A.N, A.D, A.H, A.W, A.C, A.ld, CB, a.tw, a.th, a.td, op.stride,
                          swz_for_bytes(CB * 2), A.vD, A.vH, A.vW));
  B200_TRY(make_act_map(&maps.dy[0], Y.hi, Y.N, Y.D, Y.H, Y.W, Y.C, Y.ld, CBN, a.tw, a.th, a.td, 1,
                        swz_for_bytes(CBN * 2), Y.vD, Y.vH, Y.vW));
  if (split) {
    B200_TRY(make_act_map(&maps.a[1], A.lo, A.N, A.D, A.H, A.W, A.C, A.ld, CB, a.tw, a.th, a.td, op.stride,
                          swz_for_bytes(CB * 2), A.vD, A.vH, A.vW));
    B200_TRY(make_act_map(&maps.dy[1], Y.lo, Y.N, Y.D, Y.H, Y.W, Y.C, Y.ld, CBN, a.tw, a.th, a.td, 1,
                          swz_for_bytes(CBN * 2), Y.vD, Y.vH, Y.vW));
  }
  const dim3 grid((unsigned)r.splits, (unsigned)r.groups, (unsigned)r.cotiles);
  return with_wgrad_kernel(r, [&](auto k) {
    return launch_wg<decltype(k)::CB, decltype(k)::BN, decltype(k)::HALO>(maps, a, grid, st);
  });
}

}  // namespace b200
