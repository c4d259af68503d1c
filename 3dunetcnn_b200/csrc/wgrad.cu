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
// Work item = (group of up to 2 * 128/BN M tiles, N tile); iteration = (work item, voxel tile).  The per-tap kernel is
// stream-K: `ctas` persistent CTAs take contiguous, equal (within one) ranges of the items x voxel tiles iterations, items
// outer, and flush their register accumulators whenever the item changes and at the end of the range.  Two consumer
// warpgroups share each dY tile, each with its own M tiles; an item with a single M tile splits its voxel tiles between them.
// Partial sums are reduced into the fp32 gradient buffer with vector atomics, or stored into the slot of the CTA's rank among
// the item's CTAs (deterministic mode).  Split-precision mode: passes (a_hi,dy_hi), (a_lo,dy_hi), (a_hi,dy_lo).  3x3x3
// stride-1 layers of at most 64 input channels run in halo mode instead (k_wgrad_halo, WgradHaloCfg: grid of splits x M-tile
// groups x N tiles).
#include <algorithm>
#include "conv_common.cuh"

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
  int qt;         // M-tiles per CTA (per-tap kernel: per work item)
  int kblocks;    // voxel tiles in total
  int splits;     // halo kernel: split-K CTAs per work item; per-tap kernel: partial slots per work item (deterministic mode)
  int cotiles;    // N tiles
  int items;      // per-tap kernel: work items, M-tile groups x cotiles
  int ctas;       // per-tap kernel: persistent CTAs over the items x kblocks iterations
  int npass;
  float* dw;
  float* part;             // deterministic mode: per-split partial sums [splits][T][Cip][Cop] (plain stores) instead of atomics
  long long part_stride;   // elements per split
};

constexpr int WG_A_STAGES = 2;   // per consumer warpgroup
constexpr int WG_D_STAGES = 2;
constexpr int WG_A_BYTES = 32768;

template <int CB, int BN>
struct WgradCfg {
  static constexpr int CBN = BN < 64 ? BN : 64;
  static constexpr int BPM = 128 / CB;             // boxes per M tile
  static constexpr int BPN = BN / CBN;             // boxes per N tile
  static constexpr int QT = 128 / BN;              // M tiles per consumer warpgroup: QT * BN fp32 accumulator registers per thread
  static constexpr int D_BYTES = BN * 128 * 2;
  static constexpr int D_STAGE = D_BYTES < 1024 ? 1024 : D_BYTES;
  static constexpr int A_REGION = 2 * WG_A_STAGES * WG_A_BYTES;   // one A ring per consumer warpgroup
  static constexpr int SMEM_BYTES = A_REGION + WG_D_STAGES * D_STAGE + 1024 + 1024;
  static_assert(SMEM_BYTES <= 232448, "wgrad: configuration does not fit shared memory");
  static constexpr uint32_t LAYOUT_A = swizzle_for_row_bytes(CB * 2);
  static constexpr uint32_t LAYOUT_B = swizzle_for_row_bytes(CBN * 2);
  static constexpr uint32_t SBO_A = 16 * CB, LBO_A = 256 * CB;
  static constexpr uint32_t SBO_B = 16 * CBN, LBO_B = 256 * CBN;
  static constexpr uint32_t HALF_M = 64 / CB * LBO_A;   // bytes from M row 0 to M row 64
};

// Halo mode (wgrad_halo_eligible): per voxel tile ONE TMA halo box of 64 channels (HaloTile; channels past the input's are the
// TMA out-of-bounds zero fill) replaces the per-tap boxes.  Each m64 half of an M tile is one tap of all 64 channels, read from the
// box at the tap's row with a K-group stride (SBO) of one halo row.  Two consumer warpgroups share every box and dY tile, each
// with its own M tiles; two stages (box + dY tile): the producer loads the next voxel tile while the MMAs of this one run.
template <int BN>
struct WgradHaloCfg : WgradCfg<64, BN> {
  static constexpr int ROWB = 128;                 // bytes per box row
  static constexpr int BOX_TX = HaloTile::ROWS * ROWB;
  static constexpr int BOX_BYTES = (BOX_TX + 1023) / 1024 * 1024;
  static constexpr int STAGES = 2;
  static constexpr int SMEM_BYTES = STAGES * (BOX_BYTES + WgradCfg<64, BN>::D_STAGE) + 1024 + 1024;
  static_assert(SMEM_BYTES <= 232448, "wgrad: configuration does not fit shared memory");
};

// Stream-K partition of the per-tap kernel: CTA c of P runs iterations [c * T / P, (c + 1) * T / P) of the T = items x kblocks,
// items outer.  The CTA that runs iteration x:
__host__ __device__ inline int wgrad_sk_cta(long long x, long long T, int P) { return (int)(((x + 1) * P - 1) / T); }

__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// Warps 0-7: two consumer warpgroups (wgmma issue and the write-back); warp 8: TMA producer.  Every CTA walks its stream-K
// range as segments of one work item each.  An item of nq >= 2 M tiles gives warpgroup 0 its first ceil(nq / 2) M tiles and
// warpgroup 1 the rest, and both read every dY tile.  An item of one M tile gives it to both: warpgroup g takes the segment's
// voxel tiles kb with (kb - kb0) % 2 == g.  Each warpgroup has its own A ring; the dY ring is released by all eight warps.
template <int CB, int BN>
__global__ void __launch_bounds__(288, 1) k_wgrad(const __grid_constant__ WgradMaps maps, const WgradArgs p) {
  using Cfg = WgradCfg<CB, BN>;
  constexpr int SA = WG_A_STAGES, SD = WG_D_STAGES;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment by pointer arithmetic on the __shared__ array: an integer round trip loses the address space and every
  // shared-memory access below would compile to a generic LD.E / ST.E instead of LDS / STS
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;   // ring of warpgroup g: stages [g * SA, (g + 1) * SA)
  uint8_t* smem_d = smem + Cfg::A_REGION;
  uint8_t* aux = smem_d + SD * Cfg::D_STAGE;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(aux);
  uint64_t* a_empty = a_full + 2 * SA;
  uint64_t* d_full = a_empty + 2 * SA;
  uint64_t* d_empty = d_full + SD;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int T = p.items * p.kblocks;
  const int it_begin = (int)((long long)T * blockIdx.x / p.ctas), it_end = (int)((long long)T * (blockIdx.x + 1) / p.ctas);

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&maps.a[0]);
    tma_prefetch_desc(&maps.dy[0]);
    for (int s = 0; s < 2 * SA; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 4); }
    for (int s = 0; s < SD; ++s) { mbar_init(&d_full[s], 1); mbar_init(&d_empty[s], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();                 // set-up above overlaps the tail of the previous kernel; no global access before this line
  pdl_launch_dependents();
  const int pad = p.pad;

  if (warp == 8) {
    const uint32_t issue = elect_one() ? 1u : 0u;
    int ia0 = 0, ia1 = 0, id = 0;
    for (int it = it_begin; it < it_end;) {
      const int item = it / p.kblocks;
      const int kb0 = it - item * p.kblocks;
      const int kb1 = min(p.kblocks, kb0 + (it_end - it));
      it += kb1 - kb0;
      const int q0 = item / p.cotiles * p.qt, co0 = item % p.cotiles * BN;
      const int nq = min(p.qt, p.qtiles - q0), n0 = (nq + 1) >> 1;
      for (int kb = kb0; kb < kb1; ++kb) {
        int t = kb;
        const int wt = t % p.tiles_w; t /= p.tiles_w;
        const int ht = t % p.tiles_h; t /= p.tiles_h;
        const int dt = t % p.tiles_d;
        const int n = t / p.tiles_d;
        const int w0 = wt * p.tw, h0 = ht * p.th, d0 = dt * p.td;
        const int own = (kb - kb0) & 1;   // single-M-tile item: the warpgroup that takes this voxel tile
        for (int pass = 0; pass < p.npass; ++pass) {
          {
            const int s = id % SD;
            const uint32_t ph = (id / SD) & 1;
            mbar_wait(&d_empty[s], ph ^ 1);
            mbar_expect_tx_if(issue, &d_full[s], Cfg::D_BYTES);
            uint8_t* dst = smem_d + s * Cfg::D_STAGE;
#pragma unroll
            for (int bx = 0; bx < Cfg::BPN; ++bx)
              tma_load_5d_if(issue, dst + bx * Cfg::LBO_B, &maps.dy[pass == 2], &d_full[s], co0 + bx * Cfg::CBN, w0, h0, d0, n);
            ++id;
          }
#pragma unroll
          for (int qi = 0; qi < Cfg::QT; ++qi) {
#pragma unroll
            for (int g = 0; g < 2; ++g) {
              int q;
              if (nq == 1) {
                if (qi != 0 || g != own) continue;
                q = q0;
              } else {
                if (qi >= (g ? nq - n0 : n0)) continue;
                q = q0 + g * n0 + qi;
              }
              int& ia = g ? ia1 : ia0;
              const int s = g * SA + ia % SA;
              const uint32_t ph = (ia / SA) & 1;
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
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  const int wg = warp >> 2;
  constexpr uint32_t hi_a = desc_hi(Cfg::SBO_A, Cfg::LAYOUT_A), hi_b = desc_hi(Cfg::SBO_B, Cfg::LAYOUT_B);
  const uint32_t a0 = smem_u32(smem_a) + wg * SA * WG_A_BYTES, d0s = smem_u32(smem_d);
  uint64_t* my_full = a_full + wg * SA;
  uint64_t* my_empty = a_empty + wg * SA;
  float acc[Cfg::QT][2][BN / 2];
#pragma unroll
  for (int qi = 0; qi < Cfg::QT; ++qi)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { acc[qi][0][i] = 0.f; acc[qi][1][i] = 0.f; }
  int ia = 0, id = 0;
  int prev_a = -1, prev_d = -1;   // ring slots the previous wgmma group read: handed back once that group has retired
  for (int it = it_begin; it < it_end;) {
    const int item = it / p.kblocks;
    const int kb0 = it - item * p.kblocks;
    const int kb1 = min(p.kblocks, kb0 + (it_end - it));
    it += kb1 - kb0;
    const int q0 = item / p.cotiles * p.qt, co0 = item % p.cotiles * BN;
    const int nq = min(p.qt, p.qtiles - q0), n0 = (nq + 1) >> 1;
    const int nt = nq == 1 ? 1 : wg ? nq - n0 : n0;   // M tiles of this warpgroup
    const int qw = nq == 1 ? q0 : q0 + wg * n0;       // its first
    for (int kb = kb0; kb < kb1; ++kb) {
      const bool mine = nq > 1 || ((kb - kb0) & 1) == wg;
      for (int pass = 0; pass < p.npass; ++pass) {
        const int sd = id % SD;
        mbar_wait(&d_full[sd], (id / SD) & 1);
        ++id;
        if (!mine) {   // the other warpgroup's voxel tile: retire this one's MMAs (the slots they hold gate the producer)
          wgmma_wait<0>();
          if (lane == 0) {
            if (prev_a >= 0) mbar_arrive(&my_empty[prev_a]);
            if (prev_d >= 0) mbar_arrive(&d_empty[prev_d]);
            mbar_arrive(&d_empty[sd]);
          }
          prev_a = prev_d = -1;
          continue;
        }
        const uint32_t b_lo = desc_lo(d0s + sd * Cfg::D_STAGE, Cfg::LBO_B);
#pragma unroll
        for (int qi = 0; qi < Cfg::QT; ++qi) {
          if (qi < nt) {
            const int sa = ia % SA;
            mbar_wait(&my_full[sa], (ia / SA) & 1);
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
              if (prev_a >= 0) mbar_arrive(&my_empty[prev_a]);
              if (prev_d >= 0) mbar_arrive(&d_empty[prev_d]);
            }
            prev_a = sa;
            prev_d = qi == nt - 1 ? sd : -1;
            ++ia;
          }
        }
      }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int qi = 0; qi < Cfg::QT; ++qi) { wgmma_fence_regs(acc[qi][0]); wgmma_fence_regs(acc[qi][1]); }
    if (lane == 0) {
      if (prev_a >= 0) mbar_arrive(&my_empty[prev_a]);
      if (prev_d >= 0) mbar_arrive(&d_empty[prev_d]);
    }
    prev_a = prev_d = -1;

    // flush the item's partial sum straight from the fragments: element (row r, column c) of M tile q -> [tap][ci][co0 + c]
    // at element offset off.  Deterministic mode: slot = the CTA's rank among the CTAs of the item; the item's last CTA also
    // zeroes the slots above its own, which no CTA of this item writes.
    int slot = 0;
    if (p.part) slot = (int)blockIdx.x - wgrad_sk_cta((long long)item * p.kblocks, T, p.ctas);
    const bool zero_rest = p.part && kb1 == p.kblocks && (nq > 1 || wg == 0);
    auto frags = [&](auto&& f) {
#pragma unroll
      for (int qi = 0; qi < Cfg::QT; ++qi) {
        if (qi >= nt) continue;
#pragma unroll
        for (int hm = 0; hm < 2; ++hm) {
#pragma unroll
          for (int r8 = 0; r8 < 2; ++r8) {
            const int row = hm * 64 + (warp & 3) * 16 + (lane >> 2) + r8 * 8;
            const int u = (qw + qi) * Cfg::BPM + row / CB;
            const int tap = u / p.nci, cic = u % p.nci;
            const int ci = cic * CB + row % CB;
            if (u >= p.units || ci >= p.Ci) continue;
            const long long off = ((long long)tap * p.Cip + ci) * p.Cop;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
              const int c = co0 + j * 8 + 2 * (lane & 3);
              if (c < p.Cop)   // Cop is a multiple of 4 and c is even: c + 1 < Cop as well
                f(off + c, make_float2(acc[qi][hm][4 * j + 2 * r8], acc[qi][hm][4 * j + 2 * r8 + 1]));
            }
          }
        }
      }
    };
    if (!p.part) {
      frags([&](long long off, float2 v) { atomicAdd(reinterpret_cast<float2*>(p.dw + off), v); });
    } else {
      float* const base = p.part + slot * p.part_stride;
      if (nq == 1) {   // both warpgroups hold a partial sum of the one M tile: warpgroup 1's, then warpgroup 0 adds its own
        if (wg == 1) frags([&](long long off, float2 v) { *reinterpret_cast<float2*>(base + off) = v; });
        named_bar_sync(1, 256);
        if (wg == 0)
          frags([&](long long off, float2 v) {
            const float2 o = __ldcg(reinterpret_cast<const float2*>(base + off));
            *reinterpret_cast<float2*>(base + off) = make_float2(o.x + v.x, o.y + v.y);
          });
      } else {
        frags([&](long long off, float2 v) { *reinterpret_cast<float2*>(base + off) = v; });
      }
      if (zero_rest)
        for (int s = slot + 1; s < p.splits; ++s)
          frags([&](long long off, float2) { *reinterpret_cast<float2*>(p.part + s * p.part_stride + off) = make_float2(0.f, 0.f); });
    }
#pragma unroll
    for (int qi = 0; qi < Cfg::QT; ++qi)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) { acc[qi][0][i] = 0.f; acc[qi][1][i] = 0.f; }
  }
}

// Halo mode (WgradHaloCfg).  Warps 0-7: two consumer warpgroups, warpgroup g owning M tiles [q0 + g * qw, q0 + (g + 1) * qw) of
// the CTA's p.qt with qw = ceil(p.qt / 2); warp 8: TMA producer.  M half hm of M tile q is tap 2q + hm; K step k = output rows
// h = 2k, 2k + 1 of the voxel tile.
template <int BN>
__global__ void __launch_bounds__(288, 1) k_wgrad_halo(const __grid_constant__ WgradMaps maps, const WgradArgs p) {
  using Cfg = WgradHaloCfg<BN>;
  constexpr int S = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // (see k_wgrad)
  uint8_t* smem_a = smem;
  uint8_t* smem_d = smem + S * Cfg::BOX_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_d + S * Cfg::D_STAGE);   // stage s: box s and dY tile s
  uint64_t* empty = full + S;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int split = blockIdx.x;
  const int q0 = blockIdx.y * p.qt;
  const int q1 = min(q0 + p.qt, p.qtiles);
  const int co0 = blockIdx.z * BN;
  const int kb0 = (int)((long long)p.kblocks * split / p.splits);
  const int kb1 = (int)((long long)p.kblocks * (split + 1) / p.splits);

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&maps.a[0]);
    tma_prefetch_desc(&maps.dy[0]);
    for (int s = 0; s < S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();                 // (see k_wgrad)
  pdl_launch_dependents();

  if (warp == 8) {
    const uint32_t issue = elect_one() ? 1u : 0u;
    for (int kb = kb0; kb < kb1; ++kb) {
      int t = kb;
      const int wt = t % p.tiles_w; t /= p.tiles_w;
      const int ht = t % p.tiles_h; t /= p.tiles_h;
      const int dt = t % p.tiles_d;
      const int n = t / p.tiles_d;
      const int w0 = wt * p.tw, h0 = ht * p.th, d0 = dt * p.td;
      const int kbi = kb - kb0, s = kbi % S;
      mbar_wait(&empty[s], ((kbi / S) & 1) ^ 1);
      mbar_expect_tx_if(issue, &full[s], Cfg::BOX_TX + Cfg::D_BYTES);
#pragma unroll
      for (int bx = 0; bx < Cfg::BPN; ++bx)
        tma_load_5d_if(issue, smem_d + s * Cfg::D_STAGE + bx * Cfg::LBO_B, &maps.dy[0], &full[s], co0 + bx * Cfg::CBN, w0, h0, d0, n);
      tma_load_5d_if(issue, smem_a + s * Cfg::BOX_BYTES, &maps.a[0], &full[s], 0, w0 - 1, h0 - 1, d0 - 1, n);
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  const int wg = warp >> 2;
  const int qw = (p.qt + 1) >> 1;
  const int qa = q0 + wg * qw;
  const int nq = min(qa + qw, q1) - qa;   // M tiles of this warpgroup (none in a last group with a single M tile)
  constexpr uint32_t hi_a = desc_hi(HaloTile::GROUP_STRIDE * Cfg::ROWB, Cfg::LAYOUT_A);
  constexpr uint32_t hi_b = desc_hi(Cfg::SBO_B, Cfg::LAYOUT_B);
  constexpr uint32_t K_STEP = 2 * HaloTile::GROUP_STRIDE * Cfg::ROWB >> 4;   // descriptor offset of the next two output rows
  // descriptor offsets of this warpgroup's M halves from the box start: the tap's first row
  uint32_t off[Cfg::QT][2];
#pragma unroll
  for (int qi = 0; qi < Cfg::QT; ++qi)
#pragma unroll
    for (int hm = 0; hm < 2; ++hm) {
      int u = 2 * (qa + qi) + hm;
      if (u >= p.units) u = p.units - 1;   // duplicate a valid tap; its rows are never written back
      off[qi][hm] = HaloTile::tap_row(u) * (Cfg::ROWB >> 4);
    }
  const uint32_t a0 = smem_u32(smem_a), d0s = smem_u32(smem_d);
  float acc[Cfg::QT][2][BN / 2];
#pragma unroll
  for (int qi = 0; qi < Cfg::QT; ++qi)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { acc[qi][0][i] = 0.f; acc[qi][1][i] = 0.f; }
  for (int kb = kb0; kb < kb1; ++kb) {
    const int kbi = kb - kb0, s = kbi % S;
    mbar_wait(&full[s], (kbi / S) & 1);
    const uint32_t a_lo = desc_lo(a0 + s * Cfg::BOX_BYTES, 16);   // (LBO unused: an m64 half is one 128-byte swizzle atom)
    const uint32_t b_lo = desc_lo(d0s + s * Cfg::D_STAGE, Cfg::LBO_B);
#pragma unroll
    for (int qi = 0; qi < Cfg::QT; ++qi) {
      if (qi < nq) {
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const uint64_t db = desc_from(b_lo + ((k * 2 * Cfg::SBO_B) >> 4), hi_b);
          Wgmma<BN>::template mma<1, 1>(acc[qi][0], desc_from(a_lo + off[qi][0] + k * K_STEP, hi_a), db, 1u);
          Wgmma<BN>::template mma<1, 1>(acc[qi][1], desc_from(a_lo + off[qi][1] + k * K_STEP, hi_a), db, 1u);
        }
        wgmma_commit();
      }
    }
    wgmma_wait<0>();   // this stage's box and dY tile are read: hand them back (the other stage is already loading)
    if (lane == 0) mbar_arrive(&empty[s]);
  }
#pragma unroll
  for (int qi = 0; qi < Cfg::QT; ++qi) { wgmma_fence_regs(acc[qi][0]); wgmma_fence_regs(acc[qi][1]); }

  // write-back straight from the fragments: row r of half hm of M tile q -> dw[2q + hm][r][co0 + c]
  const bool has_work = kb1 > kb0;
  float* const base = p.part ? p.part + (long long)split * p.part_stride : p.dw;
#pragma unroll
  for (int qi = 0; qi < Cfg::QT; ++qi) {
    if (qi >= nq) continue;
#pragma unroll
    for (int hm = 0; hm < 2; ++hm) {
#pragma unroll
      for (int r8 = 0; r8 < 2; ++r8) {
        const int row = (warp & 3) * 16 + (lane >> 2) + r8 * 8;
        const int tap = 2 * (qa + qi) + hm, ci = row;
        if (tap >= p.units || ci >= p.Ci || !(has_work || p.part)) continue;
        float* dst = base + ((long long)tap * p.Cip + ci) * p.Cop;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = co0 + j * 8 + 2 * (lane & 3);
          if (c < p.Cop) {   // (see k_wgrad)
            const float2 v = make_float2(acc[qi][hm][4 * j + 2 * r8], acc[qi][hm][4 * j + 2 * r8 + 1]);
            if (p.part) *reinterpret_cast<float2*>(dst + c) = has_work ? v : make_float2(0.f, 0.f);
            else atomicAdd(reinterpret_cast<float2*>(dst + c), v);
          }
        }
      }
    }
  }
}

template <int CB, int BN, bool HALO>
static int launch_wg(const WgradMaps& maps, const WgradArgs& a, dim3 grid, cudaStream_t st) {
  if constexpr (HALO) {
    static_assert(CB == 64, "halo mode loads 64-channel boxes");
    using Cfg = WgradHaloCfg<BN>;
    B200_TRY((set_max_dynamic_smem<k_wgrad_halo<BN>>(Cfg::SMEM_BYTES)));
    launch_pdl(k_wgrad_halo<BN>, grid, dim3(288), Cfg::SMEM_BYTES, st, maps, a);
  } else {
    using Cfg = WgradCfg<CB, BN>;
    B200_TRY((set_max_dynamic_smem<k_wgrad<CB, BN>>(Cfg::SMEM_BYTES)));
    launch_pdl(k_wgrad<CB, BN>, grid, dim3(288), Cfg::SMEM_BYTES, st, maps, a);
  }
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// Halo mode (see WgradHaloCfg): 3x3x3 stride 1, bf16, output planes filling the 8 x 16 halo tile, 33..64 input channels -- and
// 8..32 input channels when BN <= 32.  On per-tap tiles every M tile of a CTA re-loads 32 KB of activation boxes per voxel tile
// for only BN columns of MMA, so at BN <= 32 those launches are bound by L2 -> shared-memory traffic; one 64-channel box per
// voxel tile, zero-filled past the input's channels, removes that traffic at the price of MMAs on the zero channels.  At BN >= 64
// the per-tap kernel is no longer bound by its A loads, and the 2-4x MMAs of the padded box would cost more than they save.
static bool wgrad_halo_eligible(const WgradOp& op) {
  const Act& A = op.a;
  const Act& Y = op.dy;
  return !halo_disabled() && op.ksz == 3 && op.stride == 1 && !op.nopad && !A.lo && !Y.lo && A.C <= 64 &&
         (A.C > 32 || bn_bucket(Y.C) <= 32) && Y.W >= HaloTile::TW && Y.H >= HaloTile::TH && A.D == Y.D && A.H == Y.H &&
         A.W == Y.W;
}

// The tiling fields of r for halo tiles or per-tap tiles: voxel tile, CB / BN, M tiles and their CTA groups (work items), N
// tiles, voxel tiles, the CTAs, the split-K factor and the partial-buffer bytes of deterministic mode.  Halo tiles: a grid of
// splits x groups x cotiles CTAs, each on one item and kblocks / splits voxel tiles.  Per-tap tiles: stream-K (k_wgrad) over
// min(num_sms, T) CTAs, T = items x kblocks; splits = the most CTAs that share one item, the partial slots it needs.
static void wgrad_tiling(const WgradOp& op, int num_sms, bool halo, WgradRoute* r) {
  const Act& A = op.a;
  const Act& Y = op.dy;
  if (halo) {
    r->tw = HaloTile::TW; r->th = HaloTile::TH; r->td = HaloTile::TD;
  } else {
    pick_tile(Y.W, Y.H, Y.D, r->tw, r->th, r->td);
  }
  const int ntaps = op.ksz * op.ksz * op.ksz;
  r->CB = halo ? 64 : kc_bucket(A.C);   // halo mode: one 64-channel box whatever the input's width
  r->BN = bn_bucket(Y.C);
  r->nci = ceil_div(A.C, r->CB);
  r->units = ntaps * r->nci;
  r->qtiles = ceil_div(r->units, 128 / r->CB);
  r->QT = 2 * (128 / r->BN);   // two consumer warpgroups of WgradCfg::QT M tiles each
  if (r->QT > r->qtiles) r->QT = r->qtiles;
  r->groups = ceil_div(r->qtiles, r->QT);
  r->QT = ceil_div(r->qtiles, r->groups);   // rebalance M tiles across groups
  r->cotiles = ceil_div(Y.C, r->BN);
  r->kblocks = Y.N * ceil_div(Y.D, r->td) * ceil_div(Y.H, r->th) * ceil_div(Y.W, r->tw);
  if (halo) {
    r->splits = num_sms / (r->groups * r->cotiles);
    if (r->splits < 1) r->splits = 1;
    if (r->splits > r->kblocks) r->splits = r->kblocks;
    r->ctas = r->splits * r->groups * r->cotiles;
  } else {
    const int items = r->groups * r->cotiles;
    const long long T = (long long)items * r->kblocks;   // < 2^31: k_wgrad counts iterations in int
    r->ctas = (int)std::min<long long>(num_sms, T);
    r->splits = 1;
    for (int i = 0; i < items; ++i)
      r->splits = std::max(r->splits, wgrad_sk_cta((long long)(i + 1) * r->kblocks - 1, T, r->ctas) -
                                          wgrad_sk_cta((long long)i * r->kblocks, T, r->ctas) + 1);
  }
  r->part_bytes = (size_t)r->splits * ntaps * op.Cip * op.Cop * sizeof(float);
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

size_t wgrad_partial_bytes(const WgradOp& op, int num_sms) {
  // both tilings: a shape-only op (no lo pointers) cannot tell whether a split-precision launch will take halo mode
  WgradRoute tap = {}, halo = {};
  wgrad_tiling(op, num_sms, false, &tap);
  if (wgrad_halo_eligible(op)) wgrad_tiling(op, num_sms, true, &halo);
  return std::max(tap.part_bytes, halo.part_bytes);
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
  wgrad_tiling(op, num_sms, halo, r);
  B200_REQUIRE((long long)r->groups * r->cotiles * r->kblocks <= INT_MAX, E_UNSUPPORTED, "wgrad: too many voxel tiles");
  r->npass = split ? 3 : 1;
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
  a.cotiles = r.cotiles;
  a.items = r.groups * r.cotiles;
  a.ctas = r.ctas;
  a.npass = r.npass;
  a.dw = op.dw;
  if (op.part) {
    a.part = op.part;
    a.part_stride = (long long)a.ntaps * op.Cip * op.Cop;
    B200_REQUIRE(r.part_bytes <= op.part_bytes, E_INVALID, "wgrad: deterministic partial buffer too small (%d splits)", r.splits);
    if (op.part_splits) *op.part_splits = r.splits;
  }
  if (halo)   // one 64-channel halo box around the voxel tile (HaloTile)
    B200_TRY(make_act_map(&maps.a[0], A.hi, A.N, A.D, A.H, A.W, A.C, A.ld, 64, HaloTile::BW, HaloTile::BH, HaloTile::BD, 1, SWZ_128,
                          A.vD, A.vH, A.vW));
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
  const dim3 grid = halo ? dim3((unsigned)r.splits, (unsigned)r.groups, (unsigned)r.cotiles) : dim3((unsigned)r.ctas);
  return with_wgrad_kernel(r, [&](auto k) {
    return launch_wg<decltype(k)::CB, decltype(k)::BN, decltype(k)::HALO>(maps, a, grid, st);
  });
}

}  // namespace b200
