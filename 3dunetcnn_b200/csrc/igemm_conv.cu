// 3-D convolution as an implicit GEMM on the sm_90a tensor cores (wgmma).
//
//   Y[v][co] = sum_{tap, ci} A[v*stride + tap - pad][ci] * Wp[tap][co][ci]          (fp32 accumulate in registers)
//
// Replaces (forward, and data-gradient with flipped/transposed packed weights):
//   nn.Conv3d k3 s1/s2 p1, bias-free    unet3d/models/pytorch/classification/resnet.py:12-17 of the reference
//   nn.Conv3d k1                        unet3d/models/pytorch/classification/resnet.py:20-22 of the reference
// GEMM view: M = 128 output voxels (one tw x th x td spatial box of one sample), N = BN output channels,
// K = taps x Cin walked in chunks of KC channels.  Per K step the producer warp issues two TMA loads:
//   A: 5-D box (KC, tw, th, td, 1) of the NDHWC activation at the tap-shifted coordinate; the zero padding of the
//      convolution is TMA out-of-bounds fill, stride-2 convolutions use the tensor map's element strides;
//   B: 3-D box (KC, BN, 1) of the packed weights [tap][co][ci].
// Both land K-major with the hardware swizzle that matches KC (128B/64B/32B) and feed wgmma.mma_async (m64nBNk16, bf16,
// fp32 accumulate) issued by one warpgroup; a STAGES-deep mbarrier ring decouples TMA from the MMAs, and a ring slot is
// handed back once the wgmma group reading it has retired.
// Epilogue (the same warpgroup, one output voxel row per thread, through an fp32 tile in shared memory) ->
//   mode 0: (+ residual) (* per-(n,c) dropout scale) -> bf16 hi[/lo] store, per-channel sum / sum-of-squares
//           for the next GroupNorm (warp butterfly -> smem -> one double atomic per channel per CTA);
//   mode 1: GroupNorm/ReLU backward: dz = dact * 1[A x + B > 0], per-channel (sum dz, sum dz*xhat).
// Split-precision ("parity") mode runs three passes per K step: Ah*Wh, Al*Wh, Ah*Wl.
#include <type_traits>
#include "conv_common.cuh"

namespace b200 {

// Kernel modes: per-tap streaming tiles, class mode (parity-class data gradient / k = s = 2 transposed convolution), and halo
// mode: the 3x3x3 stride-1 source, one K chunk wide, is loaded as ONE halo box around the output tile (HaloTile), and the 27
// taps read it through shifted shared-memory descriptors (27x less activation traffic from L2 than per-tap boxes).
// CONV_HALO_WS is halo mode on the persistent, weight-stationary kernel (k_igemm_conv_halo_ws) for the (BN, KC) whose 27 weight
// tiles fit in shared memory beside the halo box; CONV_HALO runs the ring kernel below for the wider ones.  CONV_HALO_PAIR
// (k_igemm_conv_halo_pair) shares resident weights and one two-plane halo box between two consumer warpgroups.  CONV_WIDE
// (k_igemm_conv_wide) runs per-tap tiles of 256 voxels on two consumer warpgroups that share each weight tile.
enum ConvMode { CONV_STREAM = 0, CONV_CLASS = 1, CONV_HALO = 2, CONV_HALO_WS = 3, CONV_HALO_PAIR = 4, CONV_WIDE = 5 };

// Tile sizes and shared-memory limits both convolution kernels derive from (BN, KC).
template <int BN, int KC>
struct ConvTileCfg {
  static constexpr int A_BYTES = 128 * KC * 2;
  static constexpr int B_BOX_BYTES = BN * KC * 2;
  static constexpr int B_BYTES = B_BOX_BYTES < 1024 ? 1024 : B_BOX_BYTES;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int ACC_LD = BN + 4;                     // floats per accumulator row: 16-byte aligned, rows on staggered banks
  static constexpr int ACC_BYTES = 128 * ACC_LD * 4;
  static constexpr int AUX_BYTES = 1024 + 4 * BN * 2 * 4 + BN * 16;  // barriers | per-warp stats | coef
  static constexpr int RB = KC * 2;                        // bytes per voxel row of an activation tile
  static constexpr int HALO_TX = HaloTile::ROWS * RB;
  static constexpr int HALO_BOX_BYTES = (HALO_TX + 1023) / 1024 * 1024;
  static constexpr int SMEM_LIMIT = 232448;                // sm_90 opt-in dynamic shared memory per block
  static constexpr int TWO_PER_SM = 115712;                // 228 KB per SM, 1 KB reserved per block
  static constexpr uint32_t LAYOUT = swizzle_for_row_bytes(KC * 2);
  static constexpr uint32_t SBO = 8 * KC * 2;
};

// Shared memory: STAGES-deep TMA ring | fp32 accumulator tile [128][BN + 4] | (class mode) output staging | (halo mode) halo box
// | aux.  Outside class mode the output staging tile reuses the ring: the CTA computes one tile, so every stage has been consumed
// when the epilogue starts.  Class mode keeps the staging tile apart because the producer is already loading the next class.
// BN <= 32 (<= 168 registers per thread, MIN_BLOCKS) sizes the ring so that two CTAs share an SM (one CTA's epilogue overlaps
// the other's MMAs) when that still leaves four stages; otherwise one CTA takes up to 227 KB.
//
// Weight-only ring (W_RING: halo mode with BN = 64, the 64 -> 64 channel layers): a tap stage fills only its weight box, so the
// ring holds W_STAGES weight boxes, and everything else lives in the halo box region, which nothing reads once the taps have
// retired (the grid is not persistent).  In turn it holds the halo box; the A tiles of the fused 1x1x1 second source, A tile s
// beside weight slot s, loaded once every warp's tap MMAs have retired (box_free); then the fp32 accumulator tile and the
// output staging tile.  (64, 64): 4 x 8,192 + 69,632 + 4,096 + 1,024 = 107,520 B, so two CTAs share an SM and one CTA's
// epilogue and second-source stall run under the other's MMAs.  (16, 64) and (32, 64) would fit as well, but their halo
// launches run on the two-plane kernel or stay on per-tap tiles, which already run them two per SM.
template <int BN, int KC, int MODE>
struct ConvCfg : ConvTileCfg<BN, KC> {
  using Tile = ConvTileCfg<BN, KC>;
  static constexpr int OUT_STAGING = 2 * 128 * BN * 2;    // hi + lo output tiles (class pairs: 256 rows of hi)
  static constexpr int ACC_R = (Tile::ACC_BYTES + 1023) / 1024 * 1024;
  static constexpr int W_STAGES = 4;
  static constexpr bool W_RING = MODE == CONV_HALO && BN == 64 && W_STAGES * Tile::A_BYTES <= Tile::HALO_BOX_BYTES &&
                                 ACC_R + OUT_STAGING <= Tile::HALO_BOX_BYTES &&
                                 W_STAGES * Tile::B_BYTES + Tile::HALO_BOX_BYTES + Tile::AUX_BYTES + 1024 <= Tile::TWO_PER_SM;
  static constexpr int STAGE_BYTES = W_RING ? Tile::B_BYTES : Tile::STAGE_BYTES;
  static constexpr int B_OFF = W_RING ? 0 : Tile::A_BYTES;   // weight box within a ring stage
  static constexpr int STG_BYTES = MODE == CONV_CLASS ? OUT_STAGING : 0;
  static constexpr int HALO_BYTES = MODE == CONV_HALO ? Tile::HALO_BOX_BYTES : 0;
  static constexpr int FIXED = (W_RING ? 0 : Tile::ACC_BYTES) + STG_BYTES + HALO_BYTES + Tile::AUX_BYTES + 1024;   // +1024 alignment slack
  // 2 x 160 threads fit the 64 K register file at <= 168 registers per thread (each SM sub-partition's 16 K registers hold
  // three of the ten warps)
  static constexpr int MIN_BLOCKS = BN <= 32 || W_RING ? 2 : 1;
  static constexpr int STAGES_2 = MIN_BLOCKS == 2 ? (Tile::TWO_PER_SM - FIXED) / STAGE_BYTES : 0;
  static constexpr int STAGES_RAW = W_RING ? W_STAGES : STAGES_2 >= 4 ? STAGES_2 : (Tile::SMEM_LIMIT - FIXED) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 6 ? 6 : STAGES_RAW;
  static constexpr int BLOCKS_PER_SM = STAGES_2 >= 4 ? 2 : 1;
  static constexpr int PIPE_BYTES = W_RING || STAGES * STAGE_BYTES > OUT_STAGING ? STAGES * STAGE_BYTES : OUT_STAGING;
  static constexpr int SMEM_BYTES = PIPE_BYTES + FIXED;
  static_assert(STAGES >= 2 && SMEM_BYTES <= Tile::SMEM_LIMIT, "igemm_conv: configuration does not fit shared memory");
  static_assert(!W_RING || (BLOCKS_PER_SM == 2 && SMEM_BYTES <= Tile::TWO_PER_SM), "igemm_conv: weight-only halo ring");
};

// Accumulator fragments of the two m64 halves -> s_acc (row-major, ACC_LD floats per row), so that each thread drains one
// output voxel row in the epilogue.
template <int BN, int ACC_LD>
__device__ __forceinline__ void store_acc(float* s_acc, const float (&acc)[2][BN / 2], int warp, int lane) {
#pragma unroll
  for (int hm = 0; hm < 2; ++hm) {
    const int r0 = hm * 64 + warp * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = j * 8 + 2 * (lane & 3);
      *reinterpret_cast<float2*>(s_acc + r0 * ACC_LD + c) = make_float2(acc[hm][4 * j], acc[hm][4 * j + 1]);
      *reinterpret_cast<float2*>(s_acc + (r0 + 8) * ACC_LD + c) = make_float2(acc[hm][4 * j + 2], acc[hm][4 * j + 3]);
    }
  }
}

// Mode 1: the norm coefficients of sample n for the N tile at n0 -> s_coef (zero beyond Cout), by the 128 threads tid of one
// consumer warpgroup.
template <int BN>
__device__ __forceinline__ void load_coef(float4* s_coef, const ConvArgs& p, int n, int n0, int tid) {
  for (int c = tid; c < BN; c += 128)
    s_coef[c] = (n0 + c < p.Cout) ? p.coef[(long long)n * p.coef_ld + n0 + c] : make_float4(0.f, 0.f, 0.f, 0.f);
}

// The epilogue warps' fp32 partial sums of sample n -> one fp64 atomic per channel statistic into dst [N][ld][2] (mode 0:
// stats, mode 1: bstats), by the 128 threads tid of the warpgroup that owns s_stats; `restart` zeroes the slots for the next tile.
template <int BN>
__device__ __forceinline__ void flush_stats(float* s_stats, double* dst, int ld, int Cout, int n, int n0, bool restart, int tid) {
  for (int c = tid; c < BN * 2; c += 128) {
    const float v = s_stats[c] + s_stats[BN * 2 + c] + s_stats[2 * BN * 2 + c] + s_stats[3 * BN * 2 + c];
    if (restart) { s_stats[c] = 0.f; s_stats[BN * 2 + c] = 0.f; s_stats[2 * BN * 2 + c] = 0.f; s_stats[3 * BN * 2 + c] = 0.f; }
    if (n0 + (c >> 1) < Cout) atomicAdd(&dst[((long long)n * ld + n0) * 2 + c], (double)v);
  }
}

// Start (descriptor units) of the A operand of tap `tap` in the halo box whose descriptor starts at box_lo.
template <int RB>
__device__ __forceinline__ uint32_t halo_tap_lo(uint32_t box_lo, int tap) {
  return box_lo + ((HaloTile::tap_row(tap) * RB) >> 4);
}

// Warps 0-3: one consumer warpgroup (wgmma issue, then the epilogue, one output voxel row per thread); warp 4: TMA producer.
template <int BN, int KC, int MODE>
__global__ void __launch_bounds__(160, (ConvCfg<BN, KC, MODE>::MIN_BLOCKS)) k_igemm_conv(const __grid_constant__ ConvMaps maps,
                                                                                       const ConvArgs p,
                                                                                       const __grid_constant__ ConvClassMaps cmaps) {
  using Cfg = ConvCfg<BN, KC, MODE>;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment by pointer arithmetic on the __shared__ array: an integer round trip loses the address space and every
  // shared-memory access below would compile to a generic LD.E / ST.E instead of LDS / STS
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* halo = smem + Cfg::PIPE_BYTES + (Cfg::W_RING ? 0 : Cfg::ACC_BYTES) + Cfg::STG_BYTES;
  float* s_acc = reinterpret_cast<float*>(Cfg::W_RING ? halo : smem + Cfg::PIPE_BYTES);
  uint8_t* stage_out = Cfg::W_RING ? halo + Cfg::ACC_R : MODE == CONV_CLASS ? smem + Cfg::PIPE_BYTES + Cfg::ACC_BYTES : smem;
  uint8_t* aux = halo + Cfg::HALO_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(aux);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;
  uint64_t* halo_full = empty_bar + Cfg::STAGES;
  uint64_t* box_free = halo_full + 1;   // W_RING: every warp's tap MMAs have retired, the box region takes second-source A tiles
  float* s_stats = reinterpret_cast<float*>(aux + 1024);             // [4 warps][BN][2]
  float4* s_coef = reinterpret_cast<float4*>(aux + 1024 + 4 * BN * 8);   // [BN]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  int t = blockIdx.x;
  const int wt = t % p.tiles_w; t /= p.tiles_w;
  const int ht = t % p.tiles_h; t /= p.tiles_h;
  const int dt = t % p.tiles_d;
  const int n = t / p.tiles_d;
  const int w0 = wt * p.tw, h0 = ht * p.th, d0 = dt * p.td;
  const int n0 = blockIdx.y * BN;

  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&maps.a[0][0]);
    tma_prefetch_desc(&maps.b[0][0]);
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }
    mbar_init(halo_full, 1);
    mbar_init(box_free, 4);
    fence_barrier_init();
  }
  pdl_wait();   // before the first global read (the coefficient table below); the barrier set-up above overlaps the previous kernel
  if (warp < 4) {
    for (int i = threadIdx.x; i < 4 * BN * 2; i += 128) s_stats[i] = 0.f;
    if (p.mode == 1) load_coef<BN>(s_coef, p, n, n0, threadIdx.x);
  }
  __syncthreads();
  pdl_launch_dependents();

  // class mode: ONE CTA computes all eight parity classes of its voxel tile (27 tap products walked class by class, each class
  // drained by the epilogue before the next one starts).  One CTA per class would spend most of its life in set-up.  Only the
  // class-mode instances compile its code: the others keep those registers.
  const bool cls_mode = MODE == CONV_CLASS && p.cls_mode != 0;
  int total_iters = (p.ntaps[0] * p.kchunks[0] + p.ntaps[1] * p.kchunks[1]) * p.npass;
  if (cls_mode) {
    total_iters = 0;
    for (int c = 0; c < 8; ++c) total_iters += (int)p.cls_n[c] * p.kchunks[0] * p.npass;
  }

  if (warp == 4) {
    // ------------------------------------------------------------------ TMA producer (convergent, one lane issues)
    const uint32_t issue = elect_one() ? 1u : 0u;
    int it = 0;
    for (int src = 0; src < 2; ++src) {
      const int nt = p.ntaps[src];
      if (nt == 0) continue;
      const int ks = p.ksz[src], pad = p.pad[src], sd = p.stride[src];
      if (MODE == CONV_HALO && src == 0) {
        // the halo box (one K chunk; its zero padding = TMA out-of-bounds fill), then the 27 taps' weight tiles
        mbar_expect_tx_if(issue, halo_full, Cfg::HALO_TX);
        tma_load_5d_if(issue, halo, &maps.a[0][0], halo_full, 0, w0 - 1, h0 - 1, d0 - 1, n);
        for (int tap = 0; tap < 27; ++tap) {
          const int s = it % Cfg::STAGES;
          mbar_wait(&empty_bar[s], ((it / Cfg::STAGES) & 1) ^ 1);
          mbar_expect_tx_if(issue, &full_bar[s], Cfg::B_BOX_BYTES);
          tma_load_3d_if(issue, smem + s * Cfg::STAGE_BYTES + Cfg::B_OFF, &maps.b[0][0], &full_bar[s], 0, n0, tap);
          ++it;
        }
        continue;
      }
      if (Cfg::W_RING) mbar_wait(box_free, 0);   // the second source's A tiles overwrite the halo box
      for (int cls = 0; cls < (cls_mode ? 8 : 1); ++cls) {
        const int ntap_loop = cls_mode ? (int)p.cls_n[cls] : nt;
        for (int ti = 0; ti < ntap_loop; ++ti) {
          int tap = ti, cw, ch, cd;
          if (cls_mode) {   // class tap list: source voxel j + delta, packed-weight tap index
            const int e = p.cls_tap[cls][ti];
            tap = e & 31;
            cw = w0 + ((e >> 5) & 1); ch = h0 + ((e >> 6) & 1); cd = d0 + ((e >> 7) & 1);
          } else {
            const int kd = tap / (ks * ks), kh = (tap / ks) % ks, kw = tap % ks;
            cw = w0 * sd + kw - pad; ch = h0 * sd + kh - pad; cd = d0 * sd + kd - pad;
          }
          for (int kc = 0; kc < p.kchunks[src]; ++kc) {
            for (int pass = 0; pass < p.npass; ++pass) {
              const int s = it % Cfg::STAGES;
              const uint32_t ph = (it / Cfg::STAGES) & 1;
              mbar_wait(&empty_bar[s], ph ^ 1);
              mbar_expect_tx_if(issue, &full_bar[s], Cfg::A_BYTES + Cfg::B_BOX_BYTES);
              uint8_t* sa = Cfg::W_RING ? halo + s * Cfg::A_BYTES : smem + s * Cfg::STAGE_BYTES;
              tma_load_5d_if(issue, sa, &maps.a[src][pass == 1], &full_bar[s], kc * KC, cw, ch, cd, n);
              tma_load_3d_if(issue, smem + s * Cfg::STAGE_BYTES + Cfg::B_OFF, &maps.b[src][pass == 2], &full_bar[s], kc * KC, n0, tap);
              ++it;
            }
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroup: wgmma, then the epilogue
  // M = 128 output voxels as two m64 halves (rows 0-63 / 64-127 of the A tile), N = BN, K = 16 per instruction.
  constexpr uint32_t hi_d = desc_hi(Cfg::SBO, Cfg::LAYOUT);
  constexpr uint32_t HALF_M = (64 * KC * 2) >> 4;   // descriptor offset of A row 64
  const uint32_t smem0 = smem_u32(smem);
  const int row = threadIdx.x;
  const int wl = row % p.tw, hl = (row / p.tw) % p.th, dl = row / (p.tw * p.th);
  const int w = w0 + wl, h = h0 + hl, d = d0 + dl;
  const bool valid = (w < p.Wo) && (h < p.Ho) && (d < p.Do);
  const bool want_stats = (p.mode == 0) ? (p.stats != nullptr) : (p.bstats != nullptr);
  const bool edge = p.zero_last && (w == p.Wo - 1 || h == p.Ho - 1 || d == p.Do - 1);
  const bool split = p.out_lo != nullptr;
  constexpr int CBO = BN < 64 ? BN : 64;
  constexpr int SROWS_BOX = 128 * CBO * 2;
  // side inputs (residual) are indexed in the OUTPUT tensor: in class mode that is voxel 2j + p of a 2x grid
  auto vox_of = [&](int cls) -> long long {
    return cls_mode
        ? (((long long)n * (2 * p.Do) + 2 * d + ((cls >> 2) & 1)) * (2 * p.Ho) + 2 * h + ((cls >> 1) & 1)) * (2 * p.Wo) + 2 * w + (cls & 1)
        : (((long long)n * p.Do + d) * p.Ho + h) * p.Wo + w;
  };
  for (int cls = 0; cls < (cls_mode ? 8 : 1); ++cls) conv_epilogue_prefetch(p, n0, BN, vox_of(cls), valid);   // -> L2 while the MMAs run

  float acc[2][BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
  // halo mode: iterations 0..26 are the taps of source 0, read from the halo box (HaloTile)
  constexpr uint32_t hi_halo = desc_hi(HaloTile::GROUP_STRIDE * Cfg::RB, Cfg::LAYOUT);
  const uint32_t halo_lo0 = desc_lo(smem_u32(halo), 16);
  if (MODE == CONV_HALO) mbar_wait(halo_full, 0);
  int it = 0;
  for (int cls = 0; cls < (cls_mode ? 8 : 1); ++cls) {
    const int n_it = cls_mode ? (int)p.cls_n[cls] * p.kchunks[0] * p.npass : total_iters;
    int prev = -1;   // ring slot whose MMAs may still be reading it
    for (int i = 0; i < n_it; ++i, ++it) {
      const int s = it % Cfg::STAGES;
      mbar_wait(&full_bar[s], (it / Cfg::STAGES) & 1);
      uint32_t a_lo = Cfg::W_RING ? halo_lo0 + ((s * Cfg::A_BYTES) >> 4) : desc_lo(smem0 + s * Cfg::STAGE_BYTES, 16);
      uint32_t a_hi = hi_d, a_half = HALF_M;
      if (MODE == CONV_HALO && i < 27) {
        a_lo = halo_tap_lo<Cfg::RB>(halo_lo0, i);
        a_hi = hi_halo;
        a_half = (HaloTile::HALF_M * Cfg::RB) >> 4;
      }
      const uint32_t b_lo = desc_lo(smem0 + s * Cfg::STAGE_BYTES + Cfg::B_OFF, 16);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < KC / 16; ++k) {
        const uint32_t accumulate = (i > 0 || k > 0) ? 1u : 0u;   // the first K step of a class overwrites the accumulator
        Wgmma<BN>::template mma<0, 0>(acc[0], desc_from(a_lo + 2 * k, a_hi), desc_from(b_lo + 2 * k, hi_d), accumulate);
        Wgmma<BN>::template mma<0, 0>(acc[1], desc_from(a_lo + a_half + 2 * k, a_hi), desc_from(b_lo + 2 * k, hi_d), accumulate);
      }
      wgmma_commit();
      wgmma_wait<1>();   // the previous stage's MMAs are complete: hand its slot back to the producer
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = s;
      if (Cfg::W_RING && i == 26 && n_it > 27) {   // the last tap: the second source's A tiles may overwrite the box once it retires
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(box_free);
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc[0]);
    wgmma_fence_regs(acc[1]);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    if (Cfg::W_RING) asm volatile("bar.sync 1, 128;" ::: "memory");   // every warp's MMAs have retired: the box region is free

    const bool pair = MODE == CONV_CLASS && p.cls_pair != 0, pair_first = pair && (cls & 1) == 0, pair_second = pair && (cls & 1) == 1;
    if (cls > 0) {
      if (!pair_second && threadIdx.x == 0) tma_store_wait_read0();    // the previous stores have read the staging tile
      asm volatile("bar.sync 1, 128;" ::: "memory");                   // and every thread has read its s_acc row
    }
    store_acc<BN, Cfg::ACC_LD>(s_acc, acc, warp, lane);
    asm volatile("bar.sync 1, 128;" ::: "memory");

    const long long vox = vox_of(cls);
    // cls_pair: classes (pd, ph, 0) and (pd, ph, 1) interleave along W in ONE staging tile of 256 rows (row = output voxel
    // (dl, hl, 2 wl + pw) of a box 2 tw wide) that is stored through the dense class-pair map after the second drain
    const int srow = pair ? (dl * p.th + hl) * (2 * p.tw) + 2 * wl + (cls & 1) : row;
    conv_epilogue_tile<BN>(p, s_acc + row * Cfg::ACC_LD, warp, lane, n, n0, vox, valid, s_stats, s_coef, want_stats, edge, stage_out,
                           srow, split);
    if (pair_first) continue;     // the other W parity fills the odd rows of the same tile
    fence_proxy_async();
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (threadIdx.x == 0) {
      if (pair) {
        tma_store_5d(&cmaps.oc[cls & 6][0], stage_out, n0, 2 * w0, h0, d0, n);
      } else {
        const CUtensorMap* mo_hi = cls_mode ? &cmaps.oc[cls][0] : &maps.o[0];
        const CUtensorMap* mo_lo = cls_mode ? &cmaps.oc[cls][1] : &maps.o[1];
#pragma unroll
        for (int cb = 0; cb < BN / CBO; ++cb) {
          if (n0 + cb * CBO < p.Cout) {
            tma_store_5d(mo_hi, stage_out + cb * SROWS_BOX, n0 + cb * CBO, w0, h0, d0, n);
            if (split) tma_store_5d(mo_lo, stage_out + 128 * BN * 2 + cb * SROWS_BOX, n0 + cb * CBO, w0, h0, d0, n);
          }
        }
      }
      tma_store_commit();
    }
  }
  if (want_stats) {
    asm volatile("bar.sync 1, 128;" ::: "memory");
    flush_stats<BN>(s_stats, (p.mode == 0) ? p.stats : p.bstats, (p.mode == 0) ? p.stats_ld : p.coef_ld, p.Cout, n, n0, false,
                    threadIdx.x);
  }
  if (threadIdx.x == 0) tma_store_wait_all();   // the staging tile must outlive the bulk store
}

// Wide per-tap mode (CONV_WIDE) for BN = 128: a 256-voxel tile, the 128-voxel tile of the kernel above doubled in depth.  Every
// tap of a 128-channel tile is 1 M MACs per K chunk, fed by a 16 KB activation box and a 16 KB weight box from L2; here one ring
// stage holds the activation box of 256 voxels and ONE weight box, and two consumer warpgroups issue their MMAs from it, warpgroup
// g on rows 128 g .. 128 g + 127 (output planes d0 + g td / 2 ..): 48 KB per 2 M MACs instead of 32 KB per 1 M.  The producer
// loop is the kernel above's (taps, K chunks, passes, then the second source); a stage goes back to it once both warpgroups'
// MMAs have retired it (eight warp arrivals).  Every output row sees the MMA order of the 128-voxel kernel, so the stored output
// is the same bit for bit, and each warpgroup flushes its own per-channel statistics as a 128-voxel CTA does.
// 384 threads: warpgroups 0 and 1 consume, warp 8 of warpgroup 2 produces.  setmaxnreg moves the registers the producer
// warpgroup does not need to the consumers (40 / 232 per thread), whose 128-float accumulator the 168 of an even split cannot
// hold next to the epilogue.
// Shared memory: STAGES-deep ring [A 256 x KC | B 128 x KC] | bf16 output staging (64 KB) | aux (barriers | per-warp stats of 8
// warps | coef).  Once both warpgroups have retired their last MMAs the ring is drained and holds their two fp32 accumulator tiles
// [128][BN + 4], so that the two epilogues run side by side.  In bf16 the staging region holds both warpgroups' hi tiles; in
// split precision it holds the hi + lo tiles of one, and warpgroup 1 writes them once warpgroup 0's TMA store has read its own.
template <int KC>
struct WideCfg : ConvTileCfg<128, KC> {
  using Tile = ConvTileCfg<128, KC>;
  static constexpr int BN = 128;
  static constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= the 64 K register file
  static constexpr int A_BYTES = 2 * Tile::A_BYTES;
  static constexpr int STAGE_BYTES = A_BYTES + Tile::B_BYTES;
  static constexpr int OUT_TILE = 128 * BN * 2;           // one bf16 output tile of a warpgroup
  static constexpr int STG_BYTES = 2 * OUT_TILE;
  static constexpr int AUX_BYTES = 1024 + 8 * BN * 2 * 4 + BN * 16;
  static constexpr int FIXED = STG_BYTES + AUX_BYTES + 1024;   // +1024 alignment slack
  static constexpr int STAGES_RAW = (Tile::SMEM_LIMIT - FIXED) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 6 ? 6 : STAGES_RAW;
  static constexpr int BLOCKS_PER_SM = 1;
  static constexpr int PIPE_BYTES = STAGES * STAGE_BYTES > 2 * Tile::ACC_BYTES ? STAGES * STAGE_BYTES : 2 * Tile::ACC_BYTES;
  static constexpr int SMEM_BYTES = PIPE_BYTES + FIXED;
  // KC 64: 3 x 49,152 (>= 2 x 67,584) + 65,536 + 11,264 + 1,024 = 225,280 B
  static_assert(STAGES >= 3 && SMEM_BYTES <= Tile::SMEM_LIMIT && 128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= 65536,
                "igemm_conv: wide per-tap configuration");
};

template <int KC>
__global__ void __launch_bounds__(384, 1) k_igemm_conv_wide(const __grid_constant__ ConvMaps maps, const ConvArgs p) {
  using Cfg = WideCfg<KC>;
  constexpr int BN = Cfg::BN;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* stg = smem + Cfg::PIPE_BYTES;
  uint8_t* aux = stg + Cfg::STG_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(aux);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;
  float* s_stats_all = reinterpret_cast<float*>(aux + 1024);               // [8 warps][BN][2]
  float4* s_coef = reinterpret_cast<float4*>(aux + 1024 + 8 * BN * 8);     // [BN]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;                       // consumer warpgroup (2: the producer)
  const int tid = threadIdx.x & 127;

  int t = blockIdx.x;
  const int wt = t % p.tiles_w; t /= p.tiles_w;
  const int ht = t % p.tiles_h; t /= p.tiles_h;
  const int dt = t % p.tiles_d;
  const int n = t / p.tiles_d;
  const int w0 = wt * p.tw, h0 = ht * p.th, d0 = dt * p.td;
  const int n0 = blockIdx.y * BN;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&maps.a[0][0]);
    tma_prefetch_desc(&maps.b[0][0]);
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    fence_barrier_init();
  }
  pdl_wait();   // before the first global read (the coefficient table below); the barrier set-up above overlaps the previous kernel
  if (wg < 2) {
    for (int i = threadIdx.x; i < 8 * BN * 2; i += 256) s_stats_all[i] = 0.f;
    if (p.mode == 1 && wg == 0) load_coef<BN>(s_coef, p, n, n0, tid);
  }
  __syncthreads();
  pdl_launch_dependents();

  const int total_iters = (p.ntaps[0] * p.kchunks[0] + p.ntaps[1] * p.kchunks[1]) * p.npass;
  if (wg == 2) {
    // ------------------------------------------------------------------ TMA producer (warp 8 convergent, one lane issues)
    setmaxnreg_dec<Cfg::PRODUCER_REGS>();
    if (warp != 8) return;
    const uint32_t issue = elect_one() ? 1u : 0u;
    int it = 0;
    for (int src = 0; src < 2; ++src) {
      const int nt = p.ntaps[src];
      const int ks = p.ksz[src], pad = p.pad[src], sd = p.stride[src];
      for (int tap = 0; tap < nt; ++tap) {
        const int kd = tap / (ks * ks), kh = (tap / ks) % ks, kw = tap % ks;
        const int cw = w0 * sd + kw - pad, ch = h0 * sd + kh - pad, cd = d0 * sd + kd - pad;
        for (int kc = 0; kc < p.kchunks[src]; ++kc) {
          for (int pass = 0; pass < p.npass; ++pass) {
            const int s = it % Cfg::STAGES;
            mbar_wait(&empty_bar[s], ((it / Cfg::STAGES) & 1) ^ 1);
            mbar_expect_tx_if(issue, &full_bar[s], Cfg::A_BYTES + Cfg::B_BOX_BYTES);
            uint8_t* sa = smem + s * Cfg::STAGE_BYTES;
            tma_load_5d_if(issue, sa, &maps.a[src][pass == 1], &full_bar[s], kc * KC, cw, ch, cd, n);
            tma_load_3d_if(issue, sa + Cfg::A_BYTES, &maps.b[src][pass == 2], &full_bar[s], kc * KC, n0, tap);
            ++it;
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups: wgmma, then the epilogue
  setmaxnreg_inc<Cfg::CONSUMER_REGS>();
  constexpr uint32_t hi_d = desc_hi(Cfg::SBO, Cfg::LAYOUT);
  constexpr uint32_t HALF_M = (64 * KC * 2) >> 4;   // descriptor offset of A row 64 of this warpgroup's rows
  const uint32_t a_wg = desc_lo(smem_u32(smem) + wg * Cfg::Tile::A_BYTES, 16);
  const uint32_t b_lo0 = desc_lo(smem_u32(smem) + Cfg::A_BYTES, 16);
  const int row = wg * 128 + tid;
  const int wl = row % p.tw, hl = (row / p.tw) % p.th, dl = row / (p.tw * p.th);
  const int w = w0 + wl, h = h0 + hl, d = d0 + dl;
  const int dw0 = d0 + wg * (p.td >> 1);   // this warpgroup's first output plane
  const bool valid = (w < p.Wo) && (h < p.Ho) && (d < p.Do);
  const bool want_stats = (p.mode == 0) ? (p.stats != nullptr) : (p.bstats != nullptr);
  const bool edge = p.zero_last && (w == p.Wo - 1 || h == p.Ho - 1 || d == p.Do - 1);
  const bool split = p.out_lo != nullptr;
  float* s_stats = s_stats_all + wg * 4 * BN * 2;   // [4 warps][BN][2]
  float* s_acc = reinterpret_cast<float*>(smem + wg * Cfg::ACC_BYTES);   // in the drained ring
  uint8_t* stage = stg + (split ? 0 : wg * Cfg::OUT_TILE);
  const long long vox = (((long long)n * p.Do + d) * p.Ho + h) * p.Wo + w;
  conv_epilogue_prefetch(p, n0, BN, vox, valid);   // -> L2 while the MMAs run
  auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); };

  float acc[2][BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
  int prev = -1;   // ring slot whose MMAs may still be reading it
  for (int it = 0; it < total_iters; ++it) {
    const int s = it % Cfg::STAGES;
    mbar_wait(&full_bar[s], (it / Cfg::STAGES) & 1);
    const uint32_t a_lo = a_wg + ((s * Cfg::STAGE_BYTES) >> 4);
    const uint32_t b_lo = b_lo0 + ((s * Cfg::STAGE_BYTES) >> 4);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KC / 16; ++k) {
      const uint32_t accumulate = (it > 0 || k > 0) ? 1u : 0u;
      Wgmma<BN>::template mma<0, 0>(acc[0], desc_from(a_lo + 2 * k, hi_d), desc_from(b_lo + 2 * k, hi_d), accumulate);
      Wgmma<BN>::template mma<0, 0>(acc[1], desc_from(a_lo + HALF_M + 2 * k, hi_d), desc_from(b_lo + 2 * k, hi_d), accumulate);
    }
    wgmma_commit();
    wgmma_wait<1>();   // the previous stage's MMAs are complete: hand its slot back to the producer
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    prev = s;
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc[0]);
  wgmma_fence_regs(acc[1]);
  if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);

  asm volatile("bar.sync 3, 256;" ::: "memory");   // both warpgroups' MMAs have retired: the ring is free
  store_acc<BN, Cfg::ACC_LD>(s_acc, acc, warp & 3, lane);
  wg_sync();
  if (split && wg == 1) asm volatile("bar.sync 4, 256;" ::: "memory");   // warpgroup 0's store has read the staging tiles
  conv_epilogue_tile<BN>(p, s_acc + tid * Cfg::ACC_LD, warp & 3, lane, n, n0, vox, valid, s_stats, s_coef, want_stats, edge, stage,
                         tid, split);
  fence_proxy_async();
  wg_sync();
  if (tid == 0 && dw0 < p.Do) {
#pragma unroll
    for (int cb = 0; cb < BN / 64; ++cb) {
      if (n0 + cb * 64 < p.Cout) {
        tma_store_5d(&maps.o[0], stage + cb * 128 * 64 * 2, n0 + cb * 64, w0, h0, dw0, n);
        if (split) tma_store_5d(&maps.o[1], stage + 128 * BN * 2 + cb * 128 * 64 * 2, n0 + cb * 64, w0, h0, dw0, n);
      }
    }
    tma_store_commit();
  }
  if (split && wg == 0) {
    if (tid == 0) tma_store_wait_read0();
    wg_sync();
    asm volatile("bar.arrive 4, 256;" ::: "memory");
  }
  if (want_stats)
    flush_stats<BN>(s_stats, (p.mode == 0) ? p.stats : p.bstats, (p.mode == 0) ? p.stats_ld : p.coef_ld, p.Cout, n, n0, false, tid);
  if (tid == 0) tma_store_wait_all();   // the staging tile must outlive the bulk store
}

// Persistent, weight-stationary halo mode.  With one CTA per 8 x 16 x 1 tile, every CTA fetched all 27 weight tiles through the
// ring for 27 short MMA batches, then drained and ran its epilogue with nothing queued behind it.  Here a CTA loads the 27 weight
// tiles of its N tile once, behind one mbarrier, and walks the voxel tiles blockIdx.x, blockIdx.x + gridDim.x, ...  Per tile only
// the halo box is loaded (into one of HALO_BUFS buffers, so that the next box loads while this tile's epilogue runs), the 27 taps
// are one run of wgmmas with one commit, and a fused 1x1x1 second source streams its A and weight tiles through a two-stage
// ring, one stage per K chunk.  The MMA order of every output row is that of the ring kernel: taps 0..26, k16 steps inside each,
// then the second-source chunks.
// Shared memory: resident weights [27][BN][KC] | region R | HALO_BUFS halo boxes | aux.  R holds, one after the other within a
// tile, the second-source ring, the fp32 accumulator tile and the bf16 output staging tile: each thread copies its accumulator row
// into registers before the staging tile overwrites it, and the producer refills the ring only once the previous tile's TMA store
// has read the staging tile (r_free).  That is what lets BN 32 / KC 32 keep two CTAs per SM.
template <int BN, int KC>
struct HaloWsCfg : ConvTileCfg<BN, KC> {
  using Tile = ConvTileCfg<BN, KC>;
  static constexpr int STAGES = 2;                          // second-source ring
  static constexpr int W_BYTES = (27 * Tile::B_BOX_BYTES + 1023) / 1024 * 1024;
  // ACC_BYTES > the 128 x BN bf16 staging tile
  static constexpr int R_RAW = STAGES * Tile::STAGE_BYTES > Tile::ACC_BYTES ? STAGES * Tile::STAGE_BYTES : Tile::ACC_BYTES;
  static constexpr int R_BYTES = (R_RAW + 1023) / 1024 * 1024;
  static constexpr int FIXED = W_BYTES + R_BYTES + Tile::AUX_BYTES + 1024;  // +1024 alignment slack
  static constexpr int BLOCKS_PER_SM = BN <= 32 ? 2 : 1;
  static constexpr int BUDGET = BLOCKS_PER_SM == 2 ? Tile::TWO_PER_SM : Tile::SMEM_LIMIT;
  static constexpr int HALO_BUFS = FIXED + 2 * Tile::HALO_BOX_BYTES <= BUDGET ? 2 : 1;
  static constexpr int SMEM_BYTES = FIXED + HALO_BUFS * Tile::HALO_BOX_BYTES;
  // BN <= 64: the accumulator row a thread holds in registers during the epilogue stays at <= 64 floats
  static constexpr bool FITS = BN <= 64 && SMEM_BYTES <= BUDGET;
};

template <int BN, int KC>
__global__ void __launch_bounds__(160, (HaloWsCfg<BN, KC>::BLOCKS_PER_SM)) k_igemm_conv_halo_ws(const __grid_constant__ ConvMaps maps,
                                                                                              const ConvArgs p) {
  using Cfg = HaloWsCfg<BN, KC>;
  static_assert(Cfg::FITS, "igemm_conv: weight-stationary halo configuration does not fit shared memory");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* wts = smem;
  uint8_t* reg = smem + Cfg::W_BYTES;
  uint8_t* halo = reg + Cfg::R_BYTES;
  uint8_t* aux = halo + Cfg::HALO_BUFS * Cfg::HALO_BOX_BYTES;
  uint64_t* w_full = reinterpret_cast<uint64_t*>(aux);
  uint64_t* halo_full = w_full + 1;               // [HALO_BUFS]
  uint64_t* halo_empty = halo_full + 2;           // [HALO_BUFS]
  uint64_t* full_bar = halo_empty + 2;            // [STAGES]
  uint64_t* empty_bar = full_bar + Cfg::STAGES;   // [STAGES]
  uint64_t* r_free = empty_bar + Cfg::STAGES;
  float* s_stats = reinterpret_cast<float*>(aux + 1024);             // [4 warps][BN][2]
  float4* s_coef = reinterpret_cast<float4*>(aux + 1024 + 4 * BN * 8);   // [BN]
  float* s_acc = reinterpret_cast<float*>(reg);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int ntiles = p.N * p.tiles_d * p.tiles_h * p.tiles_w;
  const int n0 = blockIdx.y * BN;
  auto tile_origin = [&](int t, int& w0, int& h0, int& d0, int& n) {
    w0 = (t % p.tiles_w) * HaloTile::TW; t /= p.tiles_w;
    h0 = (t % p.tiles_h) * HaloTile::TH; t /= p.tiles_h;
    d0 = (t % p.tiles_d) * HaloTile::TD;
    n = t / p.tiles_d;
  };

  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&maps.a[0][0]);
    tma_prefetch_desc(&maps.b[0][0]);
    mbar_init(w_full, 1);
    for (int b = 0; b < Cfg::HALO_BUFS; ++b) { mbar_init(&halo_full[b], 1); mbar_init(&halo_empty[b], 4); }
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }
    mbar_init(r_free, 1);
    fence_barrier_init();
  }
  pdl_wait();   // before the first global read; the barrier set-up above overlaps the previous kernel
  if (warp < 4)
    for (int i = threadIdx.x; i < 4 * BN * 2; i += 128) s_stats[i] = 0.f;
  __syncthreads();
  pdl_launch_dependents();

  if (warp == 4) {
    // ------------------------------------------------------------------ TMA producer (convergent, one lane issues)
    const uint32_t issue = elect_one() ? 1u : 0u;
    mbar_expect_tx_if(issue, w_full, 27 * Cfg::B_BOX_BYTES);
    for (int tap = 0; tap < 27; ++tap) tma_load_3d_if(issue, wts + tap * Cfg::B_BOX_BYTES, &maps.b[0][0], w_full, 0, n0, tap);
    int it = 0, j = 0;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++j) {
      int w0, h0, d0, n;
      tile_origin(t, w0, h0, d0, n);
      const int hb = j % Cfg::HALO_BUFS;
      mbar_wait(&halo_empty[hb], ((j / Cfg::HALO_BUFS) & 1) ^ 1);
      mbar_expect_tx_if(issue, &halo_full[hb], Cfg::HALO_TX);
      tma_load_5d_if(issue, halo + hb * Cfg::HALO_BOX_BYTES, &maps.a[0][0], &halo_full[hb], 0, w0 - 1, h0 - 1, d0 - 1, n);
      if (p.ntaps[1] == 0) continue;
      mbar_wait(r_free, (j & 1) ^ 1);   // the previous tile's store has read R
      for (int kc = 0; kc < p.kchunks[1]; ++kc, ++it) {
        const int s = it % Cfg::STAGES;
        mbar_wait(&empty_bar[s], ((it / Cfg::STAGES) & 1) ^ 1);
        mbar_expect_tx_if(issue, &full_bar[s], Cfg::A_BYTES + Cfg::B_BOX_BYTES);
        uint8_t* sa = reg + s * Cfg::STAGE_BYTES;
        tma_load_5d_if(issue, sa, &maps.a[1][0], &full_bar[s], kc * KC, w0, h0, d0, n);
        tma_load_3d_if(issue, sa + Cfg::A_BYTES, &maps.b[1][0], &full_bar[s], kc * KC, n0, 0);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroup: wgmma, then the epilogue
  constexpr uint32_t hi_d = desc_hi(Cfg::SBO, Cfg::LAYOUT);
  constexpr uint32_t hi_halo = desc_hi(HaloTile::GROUP_STRIDE * Cfg::RB, Cfg::LAYOUT);
  constexpr uint32_t HALF_M = (64 * KC * 2) >> 4;                         // ring A tile: row 64
  constexpr uint32_t HALO_HALF = (HaloTile::HALF_M * Cfg::RB) >> 4;      // halo: output rows 64-127
  const uint32_t w_lo0 = desc_lo(smem_u32(wts), 16);
  const uint32_t halo_lo0 = desc_lo(smem_u32(halo), 16);
  const uint32_t reg0 = smem_u32(reg);
  const int row = threadIdx.x;
  const int wl = row % HaloTile::TW, hl = row / HaloTile::TW;
  const bool want_stats = (p.mode == 0) ? (p.stats != nullptr) : (p.bstats != nullptr);
  double* stats_dst = (p.mode == 0) ? p.stats : p.bstats;
  const int stats_ld = (p.mode == 0) ? p.stats_ld : p.coef_ld;
  int it = 0, j = 0, coef_n = -1;
  mbar_wait(w_full, 0);
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++j) {
    int w0, h0, d0, n;
    tile_origin(t, w0, h0, d0, n);
    const int w = w0 + wl, h = h0 + hl, d = d0;
    const bool valid = (w < p.Wo) && (h < p.Ho) && (d < p.Do);
    const bool edge = p.zero_last && (w == p.Wo - 1 || h == p.Ho - 1 || d == p.Do - 1);
    const long long vox = (((long long)n * p.Do + d) * p.Ho + h) * p.Wo + w;
    conv_epilogue_prefetch(p, n0, BN, vox, valid);   // -> L2 while the MMAs run

    const int hb = j % Cfg::HALO_BUFS;
    const uint32_t hlo = halo_lo0 + ((hb * Cfg::HALO_BOX_BYTES) >> 4);
    float acc[2][BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    mbar_wait(&halo_full[hb], (j / Cfg::HALO_BUFS) & 1);
    wgmma_fence();
#pragma unroll
    for (int tap = 0; tap < 27; ++tap) {
      const uint32_t a_lo = halo_tap_lo<Cfg::RB>(hlo, tap);
      const uint32_t b_lo = w_lo0 + ((tap * Cfg::B_BOX_BYTES) >> 4);
#pragma unroll
      for (int k = 0; k < KC / 16; ++k) {
        const uint32_t accumulate = (tap > 0 || k > 0) ? 1u : 0u;
        Wgmma<BN>::template mma<0, 0>(acc[0], desc_from(a_lo + 2 * k, hi_halo), desc_from(b_lo + 2 * k, hi_d), accumulate);
        Wgmma<BN>::template mma<0, 0>(acc[1], desc_from(a_lo + HALO_HALF + 2 * k, hi_halo), desc_from(b_lo + 2 * k, hi_d), accumulate);
      }
    }
    wgmma_commit();
    // while the taps run: once the previous tile's store has read R, the producer may refill it with this tile's ring stages
    if (j > 0 && threadIdx.x == 0) {
      tma_store_wait_read0();
      mbar_arrive(r_free);
    }
    int prev = -1;   // ring slot whose MMAs may still be reading it (-1: the halo box)
    for (int kc = 0; kc < p.kchunks[1]; ++kc, ++it) {
      const int s = it % Cfg::STAGES;
      mbar_wait(&full_bar[s], (it / Cfg::STAGES) & 1);
      const uint32_t a_lo = desc_lo(reg0 + s * Cfg::STAGE_BYTES, 16);
      const uint32_t b_lo = desc_lo(reg0 + s * Cfg::STAGE_BYTES + Cfg::A_BYTES, 16);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < KC / 16; ++k) {
        Wgmma<BN>::template mma<0, 0>(acc[0], desc_from(a_lo + 2 * k, hi_d), desc_from(b_lo + 2 * k, hi_d), 1u);
        Wgmma<BN>::template mma<0, 0>(acc[1], desc_from(a_lo + HALF_M + 2 * k, hi_d), desc_from(b_lo + 2 * k, hi_d), 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();   // everything before this chunk has retired: hand back the halo box or the previous ring slot
      if (lane == 0) mbar_arrive(prev < 0 ? &halo_empty[hb] : &empty_bar[prev]);
      prev = s;
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc[0]);
    wgmma_fence_regs(acc[1]);
    if (lane == 0) mbar_arrive(prev < 0 ? &halo_empty[hb] : &empty_bar[prev]);

    // every warp's MMAs have retired (the ring lived in R) and the previous store has read R
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (p.mode == 1 && n != coef_n) {   // the previous epilogue's reads of s_coef ended before its last barrier
      load_coef<BN>(s_coef, p, n, n0, threadIdx.x);
      coef_n = n;
    }
    store_acc<BN, Cfg::ACC_LD>(s_acc, acc, warp, lane);
    asm volatile("bar.sync 1, 128;" ::: "memory");
    float4 acc_row[BN / 4];
#pragma unroll
    for (int i = 0; i < BN / 4; ++i) acc_row[i] = reinterpret_cast<const float4*>(s_acc + row * Cfg::ACC_LD)[i];
    asm volatile("bar.sync 1, 128;" ::: "memory");   // the staging tile below overwrites the accumulator tile
    conv_epilogue_tile<BN>(p, reinterpret_cast<const float*>(acc_row), warp, lane, n, n0, vox, valid, s_stats, s_coef, want_stats,
                           edge, reg, row, false);
    fence_proxy_async();
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (threadIdx.x == 0) {
      tma_store_5d(&maps.o[0], reg, n0, w0, h0, d0, n);
      tma_store_commit();
    }
    if (want_stats) flush_stats<BN>(s_stats, stats_dst, stats_ld, p.Cout, n, n0, true, threadIdx.x);   // the slots restart from zero
  }
  if (threadIdx.x == 0) tma_store_wait_all();   // the staging tile must outlive the bulk store
}

// Two-plane halo mode, for the (BN, KC) whose 27 resident weight tiles take 27 x 2048 x 2 = 110,592 B: beside a halo box they
// do not fit in half the SM's shared memory, so the weight-stationary kernel runs them at one CTA per SM (whose single warpgroup
// leaves the tensor cores idle through its epilogue) and per-tap tiles reload every tap's box from L2.  Here one CTA per SM runs
// two consumer warpgroups and a TMA producer warp.  A unit of work is two 8 x 16 x 1 output tiles in consecutive planes of one
// sample; the producer loads ONE halo box (KC, 10, 18, 4) per unit, and warpgroup g computes output plane d0 + g from the box's
// plane g on (HaloBox<2>), taps 0..26 with the k16 steps inside each, as the other kernels.  Both warpgroups' MMAs share the
// resident weights; the next unit's box loads once both have retired theirs, under the two epilogues.  The epilogues take turns
// on one region R (fp32 accumulator tile, then the bf16 staging tile): warpgroup 0 first, and R passes to the other warpgroup once
// the TMA store has read it.
// Shared memory: resident weights [27][BN][KC] | halo box | R | aux (barriers | per-warp stats of 8 warps | coef per warpgroup).
template <int BN, int KC>
struct HaloPairCfg : ConvTileCfg<BN, KC> {
  using Tile = ConvTileCfg<BN, KC>;
  using Box = HaloBox<2>;
  static constexpr bool APPLIES = BN * KC == 2048 && BN <= 64;
  static constexpr int STAGES = 2;                          // output tiles in flight per unit: one per consumer warpgroup
  static constexpr int BLOCKS_PER_SM = 1;
  static constexpr int W_BYTES = (27 * Tile::B_BOX_BYTES + 1023) / 1024 * 1024;
  static constexpr int BOX_TX = Box::ROWS * Tile::RB;
  static constexpr int BOX_BYTES = (BOX_TX + 1023) / 1024 * 1024;
  static constexpr int ACC_R = (Tile::ACC_BYTES + 1023) / 1024 * 1024;   // > the 128 x BN bf16 staging tile
  static constexpr int STG_BYTES = 128 * BN * 2;
  static constexpr int AUX_BYTES = 1024 + 8 * BN * 2 * 4 + 2 * BN * 16;
  static constexpr int FIXED = W_BYTES + BOX_BYTES + ACC_R + AUX_BYTES + 1024;   // +1024 alignment slack
  // The staging tile follows the accumulator tile in R where it fits.  Otherwise it overwrites the accumulator tile, and each
  // thread first copies its accumulator row into registers: 64 more registers per thread, which BN = 64 does not have at
  // 288 threads (168 per thread).
  static constexpr bool STG_APART = FIXED + STG_BYTES <= Tile::SMEM_LIMIT;
  static constexpr int R_BYTES = ACC_R + (STG_APART ? STG_BYTES : 0);
  static constexpr int SMEM_BYTES = FIXED + (STG_APART ? STG_BYTES : 0);
  // (32, 64): 110,592 + 92,160 + 18,432 + 4,096 + 1,024 = 226,304 B, staging in the accumulator tile; (64, 32): 110,592 +
  // 46,080 + 34,816 + 16,384 + 7,168 + 1,024 = 216,064 B.  A second region R (one per warpgroup) or a second box does not fit.
  static_assert(!APPLIES || (SMEM_BYTES <= Tile::SMEM_LIMIT && (BN <= 32 || STG_APART) && SMEM_BYTES + R_BYTES > Tile::SMEM_LIMIT &&
                             SMEM_BYTES + BOX_BYTES > Tile::SMEM_LIMIT),
                "igemm_conv: two-plane halo layout");
};

template <int BN, int KC>
__global__ void __launch_bounds__(288, 1) k_igemm_conv_halo_pair(const __grid_constant__ ConvMaps maps, const ConvArgs p) {
  using Cfg = HaloPairCfg<BN, KC>;
  using Box = typename Cfg::Box;
  static_assert(Cfg::APPLIES, "igemm_conv: no two-plane halo configuration");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* wts = smem;
  uint8_t* box = smem + Cfg::W_BYTES;
  uint8_t* reg = box + Cfg::BOX_BYTES;
  uint8_t* aux = reg + Cfg::R_BYTES;
  uint64_t* w_full = reinterpret_cast<uint64_t*>(aux);
  uint64_t* box_full = w_full + 1;
  uint64_t* box_empty = w_full + 2;
  uint64_t* turn = w_full + 3;                    // [2]: warpgroup g may use R once turn[g] has completed its phase
  float* s_stats_all = reinterpret_cast<float*>(aux + 1024);   // [8 warps][BN][2]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;                       // consumer warpgroup (2: the producer warp)
  const int tid = threadIdx.x & 127;
  const int pairs_d = (p.tiles_d + 1) >> 1;
  const int nunits = p.N * pairs_d * p.tiles_h * p.tiles_w;
  const int n0 = blockIdx.y * BN;
  auto unit_origin = [&](int u, int& w0, int& h0, int& d0, int& n) {
    w0 = (u % p.tiles_w) * Box::TW; u /= p.tiles_w;
    h0 = (u % p.tiles_h) * Box::TH; u /= p.tiles_h;
    d0 = (u % pairs_d) * Box::TD;
    n = u / pairs_d;
  };

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&maps.a[0][0]);
    tma_prefetch_desc(&maps.b[0][0]);
    mbar_init(w_full, 1);
    mbar_init(box_full, 1);
    mbar_init(box_empty, 8);
    mbar_init(&turn[0], 1);
    mbar_init(&turn[1], 1);
    fence_barrier_init();
  }
  pdl_wait();   // before the first global read; the barrier set-up above overlaps the previous kernel
  if (warp < 8)
    for (int i = threadIdx.x; i < 8 * BN * 2; i += 256) s_stats_all[i] = 0.f;
  __syncthreads();
  pdl_launch_dependents();

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer (convergent, one lane issues)
    const uint32_t issue = elect_one() ? 1u : 0u;
    mbar_expect_tx_if(issue, w_full, 27 * Cfg::B_BOX_BYTES);
    for (int tap = 0; tap < 27; ++tap) tma_load_3d_if(issue, wts + tap * Cfg::B_BOX_BYTES, &maps.b[0][0], w_full, 0, n0, tap);
    int j = 0;
    for (int u = blockIdx.x; u < nunits; u += gridDim.x, ++j) {
      int w0, h0, d0, n;
      unit_origin(u, w0, h0, d0, n);
      mbar_wait(box_empty, (j & 1) ^ 1);   // both warpgroups' MMAs on the previous box have retired
      mbar_expect_tx_if(issue, box_full, Cfg::BOX_TX);
      tma_load_5d_if(issue, box, &maps.a[0][0], box_full, 0, w0 - 1, h0 - 1, d0 - 1, n);
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups: wgmma, then the epilogue
  float* s_stats = s_stats_all + wg * 4 * BN * 2;                                        // [4 warps][BN][2]
  float4* s_coef = reinterpret_cast<float4*>(aux + 1024 + 8 * BN * 8) + wg * BN;        // [BN]
  float* s_acc = reinterpret_cast<float*>(reg);
  uint8_t* stage = Cfg::STG_APART ? reg + Cfg::ACC_R : reg;
  constexpr uint32_t hi_d = desc_hi(Cfg::SBO, Cfg::LAYOUT);
  constexpr uint32_t hi_halo = desc_hi(Box::GROUP_STRIDE * Cfg::RB, Cfg::LAYOUT);
  constexpr uint32_t HALO_HALF = (Box::HALF_M * Cfg::RB) >> 4;   // halo: output rows 64-127
  const uint32_t w_lo0 = desc_lo(smem_u32(wts), 16);
  const uint32_t plane_lo = desc_lo(smem_u32(box), 16) + ((wg * Box::PLANE * Cfg::RB) >> 4);   // this warpgroup's output plane
  const int row = tid;
  const int wl = row % Box::TW, hl = row / Box::TW;
  const bool want_stats = (p.mode == 0) ? (p.stats != nullptr) : (p.bstats != nullptr);
  double* stats_dst = (p.mode == 0) ? p.stats : p.bstats;
  const int stats_ld = (p.mode == 0) ? p.stats_ld : p.coef_ld;
  auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); };
  int j = 0, coef_n = -1;
  mbar_wait(w_full, 0);
  for (int u = blockIdx.x; u < nunits; u += gridDim.x, ++j) {
    int w0, h0, d0, n;
    unit_origin(u, w0, h0, d0, n);
    const int w = w0 + wl, h = h0 + hl, d = d0 + wg;   // an odd Do leaves the second plane of the last pair outside: masked
    const bool valid = (w < p.Wo) && (h < p.Ho) && (d < p.Do);
    const bool edge = p.zero_last && (w == p.Wo - 1 || h == p.Ho - 1 || d == p.Do - 1);
    const long long vox = (((long long)n * p.Do + d) * p.Ho + h) * p.Wo + w;
    conv_epilogue_prefetch(p, n0, BN, vox, valid);   // -> L2 while the MMAs run

    float acc[2][BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    mbar_wait(box_full, j & 1);
    wgmma_fence();
#pragma unroll
    for (int tap = 0; tap < 27; ++tap) {
      const uint32_t a_lo = halo_tap_lo<Cfg::RB>(plane_lo, tap);
      const uint32_t b_lo = w_lo0 + ((tap * Cfg::B_BOX_BYTES) >> 4);
#pragma unroll
      for (int k = 0; k < KC / 16; ++k) {
        const uint32_t accumulate = (tap > 0 || k > 0) ? 1u : 0u;
        Wgmma<BN>::template mma<0, 0>(acc[0], desc_from(a_lo + 2 * k, hi_halo), desc_from(b_lo + 2 * k, hi_d), accumulate);
        Wgmma<BN>::template mma<0, 0>(acc[1], desc_from(a_lo + HALO_HALF + 2 * k, hi_halo), desc_from(b_lo + 2 * k, hi_d), accumulate);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(acc[0]);
    wgmma_fence_regs(acc[1]);
    if (lane == 0) mbar_arrive(box_empty);

    // R: warpgroup 0 takes it first in every unit (its first wait passes on the fresh barrier), warpgroup 1 after it
    mbar_wait(&turn[wg], (j & 1) ^ (wg == 0 ? 1 : 0));
    if (p.mode == 1 && n != coef_n) {   // this warpgroup's previous epilogue read s_coef before its last barrier
      load_coef<BN>(s_coef, p, n, n0, tid);
      coef_n = n;
    }
    store_acc<BN, Cfg::ACC_LD>(s_acc, acc, warp & 3, lane);
    wg_sync();
    if constexpr (Cfg::STG_APART) {
      conv_epilogue_tile<BN>(p, s_acc + row * Cfg::ACC_LD, warp & 3, lane, n, n0, vox, valid, s_stats, s_coef, want_stats, edge,
                             stage, row, false);
    } else {
      float4 acc_row[BN / 4];
#pragma unroll
      for (int i = 0; i < BN / 4; ++i) acc_row[i] = reinterpret_cast<const float4*>(s_acc + row * Cfg::ACC_LD)[i];
      wg_sync();   // the staging tile below overwrites the accumulator tile
      conv_epilogue_tile<BN>(p, reinterpret_cast<const float*>(acc_row), warp & 3, lane, n, n0, vox, valid, s_stats, s_coef,
                             want_stats, edge, stage, row, false);
    }
    fence_proxy_async();
    wg_sync();
    if (tid == 0) {
      if (d < p.Do) {
        tma_store_5d(&maps.o[0], stage, n0, w0, h0, d, n);
        tma_store_commit();
        tma_store_wait_read0();   // the store has read R: the other warpgroup may overwrite it
      }
      mbar_arrive(&turn[wg ^ 1]);
    }
    if (want_stats) flush_stats<BN>(s_stats, stats_dst, stats_ld, p.Cout, n, n0, true, tid);   // the slots restart from zero
  }
  if (tid == 0) tma_store_wait_all();
}

// ----------------------------------------------------------------------------------------------- host side
// The compile-time configuration of the kernel a (BN, KC, MODE) launch runs.
template <int BN, int KC, int MODE>
using ConvCfgOf = std::conditional_t<
    MODE == CONV_HALO_WS, HaloWsCfg<BN, KC>,
    std::conditional_t<MODE == CONV_HALO_PAIR, HaloPairCfg<BN, KC>, std::conditional_t<MODE == CONV_WIDE, WideCfg<KC>, ConvCfg<BN, KC, MODE>>>>;

template <int BN, int KC, int MODE>
static int launch_cfg(const ConvMaps& maps, const ConvArgs& args, dim3 grid, cudaStream_t st, const ConvClassMaps& cmaps) {
  using Cfg = ConvCfgOf<BN, KC, MODE>;
  if constexpr (MODE == CONV_WIDE) {
    B200_TRY((set_max_dynamic_smem<k_igemm_conv_wide<KC>>(Cfg::SMEM_BYTES)));
    launch_pdl(k_igemm_conv_wide<KC>, grid, dim3(384), Cfg::SMEM_BYTES, st, maps, args);
  } else if constexpr (MODE == CONV_HALO_PAIR) {
    B200_TRY((set_max_dynamic_smem<k_igemm_conv_halo_pair<BN, KC>>(Cfg::SMEM_BYTES)));
    launch_pdl(k_igemm_conv_halo_pair<BN, KC>, grid, dim3(288), Cfg::SMEM_BYTES, st, maps, args);
  } else if constexpr (MODE == CONV_HALO_WS) {
    B200_TRY((set_max_dynamic_smem<k_igemm_conv_halo_ws<BN, KC>>(Cfg::SMEM_BYTES)));
    launch_pdl(k_igemm_conv_halo_ws<BN, KC>, grid, dim3(160), Cfg::SMEM_BYTES, st, maps, args);
  } else {
    B200_TRY((set_max_dynamic_smem<k_igemm_conv<BN, KC, MODE>>(Cfg::SMEM_BYTES)));
    launch_pdl(k_igemm_conv<BN, KC, MODE>, grid, dim3(160), Cfg::SMEM_BYTES, st, maps, args, cmaps);
  }
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// Every (BN, KC) the dispatch below instantiates.
#define B200_CONV_CONFIGS(X)                                                                                   \
  X(16, 16) X(16, 32) X(16, 64) X(32, 16) X(32, 32) X(32, 64) X(64, 16) X(64, 32) X(64, 64) X(128, 16) X(128, 32) X(128, 64)

// KC follows the widest source among those with the largest kernel.  A fused 1x1x1 second source that is wider than the
// 3x3x3 first source is walked in more K chunks instead: sizing KC to it would pad every one of the 27 taps of the first
// source with zero channels (the 32-channel last decoder conv with its 64-channel `sample` ran at the cost of a 64-channel
// convolution).  In single-pass bf16 the nonzero products accumulate in the same order either way, so the output is the
// same bit for bit.
static int conv_kc(const ConvOp& op) {
  int k = 0;
  for (int s = 1; s < op.nsrc; ++s)
    if (op.src[s].ksz > op.src[k].ksz || (op.src[s].ksz == op.src[k].ksz && op.src[s].x.C > op.src[k].x.C)) k = s;
  return kc_bucket(op.src[k].x.C);
}

static int conv_bn(const ConvOp& op) {
  const int BN = bn_bucket(op.out.C);
  return op.cls_mode && BN > 64 ? 64 : BN;   // class mode keeps its staging tile beside the accumulator tile (ConvCfg)
}

// Halo mode runs on the weight-stationary kernel wherever its configuration fits (BN <= 64 with KC <= 32; the 27 weight tiles
// of KC = 64 or BN = 128 with KC = 32 take 221 KB), and on the ring kernel otherwise.
template <int BN, int KC>
constexpr int halo_mode() {
  return HaloWsCfg<BN, KC>::FITS ? CONV_HALO_WS : CONV_HALO;
}

// Halo mode must not cost a configuration the second CTA per SM that per-tap tiles give it.  With KC = 64 and BN <= 32 the
// halo box leaves room for fewer than four ring stages in half of the SM's shared memory; at one CTA per SM the 64 -> 32
// channel convolutions of the C2 step (forward at 128^3, data gradient at 64^3) took 1.4x as long as on per-tap tiles at
// two (H100 80GB HBM3, 400 W).  With a single K chunk per source the two modes accumulate in the same order.
template <int BN, int KC>
constexpr bool halo_keeps_occupancy() {
  return ConvCfgOf<BN, KC, halo_mode<BN, KC>()>::BLOCKS_PER_SM >= ConvCfg<BN, KC, CONV_STREAM>::BLOCKS_PER_SM;
}

static bool halo_keeps_occupancy(int BN, int KC) {
#define B200_HALO_OCC(bn, kc) \
  if (BN == bn && KC == kc) return halo_keeps_occupancy<bn, kc>();
  B200_CONV_CONFIGS(B200_HALO_OCC)
#undef B200_HALO_OCC
  return false;
}

static bool halo_pair_applies(int BN, int KC) {
#define B200_HALO_PAIR(bn, kc) \
  if (BN == bn && KC == kc) return HaloPairCfg<bn, kc>::APPLIES;
  B200_CONV_CONFIGS(B200_HALO_PAIR)
#undef B200_HALO_PAIR
  return false;
}

// Two-plane halo mode (k_igemm_conv_halo_pair) for a halo-eligible op of its (BN, KC) with one source, when its units of two
// output planes give every SM at least one: below that, pairing the tiles would leave SMs idle that the per-tile kernels use.
static bool conv_halo_pair(const ConvOp& op, int num_sms) {
  if (op.nsrc != 1 || !halo_pair_applies(conv_bn(op), conv_kc(op))) return false;
  const long long units = (long long)op.out.N * ceil_div(op.out.D, 2) * ceil_div(op.out.H, HaloTile::TH) * ceil_div(op.out.W, HaloTile::TW);
  return units * ceil_div(op.out.C, conv_bn(op)) >= num_sms;
}

// Halo mode (see ConvMode) for 3x3x3 stride-1 convolutions with <= 64 input channels (plus an optional fused 1x1x1 source)
// whose output planes fill the halo tile, in single-pass bf16, when it keeps the configuration's CTAs per SM or runs in
// two-plane halo mode.  Wider inputs stay on per-tap tiles: several halo boxes per tile were slower in the forward convolutions
// of the C2 step on the H100.
static bool conv_halo_eligible(const ConvOp& op, int num_sms) {
  if (halo_disabled() || op.cls_mode) return false;
  const ConvSrc& c = op.src[0];
  if (c.ksz != 3 || c.stride != 1 || c.nopad || c.x.C > 64) return false;
  if (op.nsrc == 2 && (op.src[1].ksz != 1 || op.src[1].stride != 1)) return false;
  for (int s = 0; s < op.nsrc; ++s)
    if (op.src[s].x.lo || op.src[s].w_lo) return false;
  if (op.out.lo) return false;   // the halo kernels store hi only; a lo output of a bf16 op runs per-tap (the epilogue splits)
  return op.out.W >= HaloTile::TW && op.out.H >= HaloTile::TH &&
         (halo_keeps_occupancy(conv_bn(op), conv_kc(op)) || conv_halo_pair(op, num_sms));
}

// The 256-voxel per-tap tile (k_igemm_conv_wide) for a BN = 128 launch whose CTAs of that tile still give every SM one: below
// that, halving the CTAs would leave SMs idle that the 128-voxel tiles use (at C2 the 16^3 launches, 64 x 2 CTAs of 128 voxels).
// tiles_hw: the (h, w) tiles of a sample, td: the depth of the 128-voxel tile.
static bool conv_wide(const ConvOp& op, int BN, int gD, int tiles_hw, int td, int num_sms) {
  if (BN != 128 || op.tile128) return false;
  return (long long)op.out.N * ceil_div(gD, 2 * td) * tiles_hw * ceil_div(op.out.C, BN) >= num_sms;
}

template <int BN_, int KC_, int MODE_>
struct ConvKernel { static constexpr int BN = BN_, KC = KC_, MODE = MODE_; };

// f(ConvKernel<BN, KC, MODE>{}) for the instantiated kernel of (kind, BN, KC) with wgs consumer warpgroups: the one selection
// conv_route reports and launch_igemm_conv launches.  E_UNSUPPORTED when no such kernel is instantiated.
template <class F>
static int with_conv_kernel(int kind, int BN, int KC, int wgs, F&& f) {
#define B200_CONV_CASE(bn, kc)                                                                              \
  if (BN == bn && KC == kc) {                                                                               \
    if (kind == CONV_KIND_CLASS1 || kind == CONV_KIND_CLASS2) {                                             \
      if constexpr (bn <= 64) return f(ConvKernel<bn, kc, CONV_CLASS>{});                                   \
    } else if (kind == CONV_KIND_HALO) {                                                                    \
      if constexpr (halo_keeps_occupancy<bn, kc>()) return f(ConvKernel<bn, kc, halo_mode<bn, kc>()>{});    \
    } else if (kind == CONV_KIND_HALO_PAIR) {                                                               \
      if constexpr (HaloPairCfg<bn, kc>::APPLIES) return f(ConvKernel<bn, kc, CONV_HALO_PAIR>{});           \
    } else if (wgs == 2) {                                                                                  \
      if constexpr (bn == 128) return f(ConvKernel<bn, kc, CONV_WIDE>{});                                   \
    } else {                                                                                                \
      return f(ConvKernel<bn, kc, CONV_STREAM>{});                                                          \
    }                                                                                                       \
  }
  B200_CONV_CONFIGS(B200_CONV_CASE)
#undef B200_CONV_CASE
  set_error("igemm_conv: no kernel for BN=%d KC=%d (kind %d, %d consumer warpgroups)", BN, KC, kind, wgs);
  return E_UNSUPPORTED;
}

int conv_route(const ConvOp& op, int num_sms, ConvRoute* r) {
  memset(r, 0, sizeof(*r));
  B200_REQUIRE(num_sms >= 1 && op.max_ctas >= 0, E_INVALID, "igemm_conv: num_sms=%d max_ctas=%d", num_sms, op.max_ctas);
  B200_REQUIRE(op.nsrc == 1 || op.nsrc == 2, E_INVALID, "igemm_conv: nsrc=%d", op.nsrc);
  B200_REQUIRE(op.cls_mode >= 0 && op.cls_mode <= 2, E_INVALID, "igemm_conv: cls_mode=%d", op.cls_mode);
  const Act& out = op.out;
  B200_REQUIRE(out.C % 8 == 0 && out.ld % 8 == 0, E_UNSUPPORTED, "igemm_conv: Cout=%d (pitch %d) must be a multiple of 8",
               out.C, out.ld);
  // class mode: the GEMM rows are the voxels of ONE parity class of the output = the source grid
  const int gD = op.cls_mode ? out.D / 2 : out.D, gH = op.cls_mode ? out.H / 2 : out.H, gW = op.cls_mode ? out.W / 2 : out.W;
  bool split = false;
  for (int s = 0; s < op.nsrc; ++s) {
    const ConvSrc& c = op.src[s];
    B200_REQUIRE(c.ksz == 1 || c.ksz == 3 || (c.ksz == 2 && c.nopad && (c.stride == 2 || op.cls_mode == 2)), E_UNSUPPORTED,
                 "igemm_conv: kernel_size=%d unsupported", c.ksz);
    B200_REQUIRE(c.stride == 1 || c.stride == 2, E_UNSUPPORTED, "igemm_conv: stride=%d unsupported", c.stride);
    B200_REQUIRE(c.x.C % 8 == 0 && c.x.ld % 8 == 0, E_UNSUPPORTED, "igemm_conv: Cin=%d must be a multiple of 8", c.x.C);
    B200_REQUIRE(c.x.N == out.N, E_INVALID, "igemm_conv: batch mismatch");
    const int pad = c.nopad ? 0 : c.ksz / 2;
    if (op.cls_mode)
      B200_REQUIRE(op.nsrc == 1 && c.ksz == (op.cls_mode == 2 ? 2 : 3) && 2 * c.x.D == out.D && 2 * c.x.H == out.H && 2 * c.x.W == out.W &&
                       op.mode == 0 && !op.bias && !op.zero_last,
                   E_INVALID, "igemm_conv: class mode needs one source at half the output extent and a plain epilogue");
    else
    B200_REQUIRE((c.x.D + 2 * pad - c.ksz) / c.stride + 1 == out.D && (c.x.H + 2 * pad - c.ksz) / c.stride + 1 == out.H &&
                     (c.x.W + 2 * pad - c.ksz) / c.stride + 1 == out.W,
                 E_INVALID, "igemm_conv: source %d dims %dx%dx%d (k%d s%d) do not produce output %dx%dx%d", s, c.x.D,
                 c.x.H, c.x.W, c.ksz, c.stride, out.D, out.H, out.W);
    if (c.x.lo || c.w_lo) split = true;
  }
  if (split) {
    for (int s = 0; s < op.nsrc; ++s)
      B200_REQUIRE(op.src[s].x.lo && op.src[s].w_lo, E_INVALID, "igemm_conv: split mode needs lo parts on every source");
    B200_REQUIRE(out.lo != nullptr, E_INVALID, "igemm_conv: split mode needs a lo output");
  }
  if (op.res) B200_REQUIRE(op.res->C == out.C, E_INVALID, "igemm_conv: residual channel mismatch");
  if (op.mode == 1) {
    B200_REQUIRE(op.gn_x && op.coef, E_INVALID, "igemm_conv: mode 1 needs gn_x and coef");
    B200_REQUIRE(op.gn_x->C == out.C, E_INVALID, "igemm_conv: gn_x channel mismatch");
  }
  const bool halo = conv_halo_eligible(op, num_sms);
  const bool pair = halo && conv_halo_pair(op, num_sms);
  r->kind = op.cls_mode == 1 ? CONV_KIND_CLASS1
          : op.cls_mode == 2 ? CONV_KIND_CLASS2
          : pair             ? CONV_KIND_HALO_PAIR
          : halo             ? CONV_KIND_HALO
                             : CONV_KIND_TAP;
  if (halo) {   // two-plane halo mode: the tile of one warpgroup (a unit of work is two tiles in consecutive planes)
    r->tw = HaloTile::TW; r->th = HaloTile::TH; r->td = HaloTile::TD;
  } else {
    pick_tile(gW, gH, gD, r->tw, r->th, r->td);
  }
  r->KC = conv_kc(op);
  r->BN = conv_bn(op);
  r->wgs = pair ? 2 : 1;
  if (r->kind == CONV_KIND_TAP && conv_wide(op, r->BN, gD, ceil_div(gH, r->th) * ceil_div(gW, r->tw), r->td, num_sms)) {
    r->td *= 2;
    r->wgs = 2;
  }
  r->tiles_w = ceil_div(gW, r->tw); r->tiles_h = ceil_div(gH, r->th); r->tiles_d = ceil_div(gD, r->td);
  for (int s = 0; s < op.nsrc; ++s) r->kchunks[s] = ceil_div(op.src[s].x.C, r->KC);
  B200_REQUIRE(!halo || r->kchunks[0] == 1, E_UNSUPPORTED, "igemm_conv: halo mode loads one K chunk of source 0 (%d)", r->kchunks[0]);
  r->npass = split ? 3 : 1;
  r->cls_pair = op.cls_mode && !split ? 1 : 0;
  r->grid[0] = (int)((long long)out.N * r->tiles_d * r->tiles_h * r->tiles_w);
  r->grid[1] = ceil_div(out.C, r->BN);
  r->grid[2] = 1;
  return with_conv_kernel(r->kind, r->BN, r->KC, r->wgs, [&](auto k) {
    using Cfg = ConvCfgOf<decltype(k)::BN, decltype(k)::KC, decltype(k)::MODE>;
    r->stages = Cfg::STAGES; r->blocks_per_sm = Cfg::BLOCKS_PER_SM; r->smem_bytes = Cfg::SMEM_BYTES;
    if constexpr (decltype(k)::MODE == CONV_HALO_WS || decltype(k)::MODE == CONV_HALO_PAIR) {
      // persistent CTAs: one wave (max_ctas, a diagnostics cap, makes small shapes walk several tiles per CTA).  In two-plane
      // mode conv_halo_pair has made sure that the wave has a unit for every CTA.
      int cap = Cfg::BLOCKS_PER_SM * num_sms / r->grid[1];
      if (cap < 1) cap = 1;
      if (op.max_ctas > 0 && op.max_ctas < cap) cap = op.max_ctas;
      if (r->grid[0] > cap) r->grid[0] = cap;
    }
    return (int)OK;
  });
}

int launch_igemm_conv(const ConvOp& op, cudaStream_t st) {
  ConvRoute r;
  B200_TRY(conv_route(op, device_sms(), &r));
  const Act& out = op.out;
  const bool pair = r.kind == CONV_KIND_HALO_PAIR;
  const bool split = r.npass == 3, halo = r.kind == CONV_KIND_HALO || pair, cls = op.cls_mode != 0;
  const bool wide = r.kind == CONV_KIND_TAP && r.wgs == 2;
  ConvArgs a;
  memset(&a, 0, sizeof(a));
  ConvMaps maps;
  memset(&maps, 0, sizeof(maps));
  a.N = out.N; a.Do = cls ? out.D / 2 : out.D; a.Ho = cls ? out.H / 2 : out.H; a.Wo = cls ? out.W / 2 : out.W; a.Cout = out.C;
  a.tw = r.tw; a.th = r.th; a.td = r.td;
  a.tiles_w = r.tiles_w; a.tiles_h = r.tiles_h; a.tiles_d = r.tiles_d;
  const int KC = r.KC;
  const int BN = r.BN;
  const Swz swz = swz_for_bytes(KC * 2);
  for (int s = 0; s < op.nsrc; ++s) {
    const ConvSrc& c = op.src[s];
    a.ntaps[s] = c.ksz * c.ksz * c.ksz; a.ksz[s] = c.ksz; a.stride[s] = c.stride; a.pad[s] = c.nopad ? 0 : c.ksz / 2;
    a.kchunks[s] = r.kchunks[s];
    const int estride = cls ? 1 : c.stride;
    const bool box = halo && s == 0;   // halo mode: source 0 is one box around the output tile (two-plane mode: the pair of tiles)
    B200_TRY(make_act_map(&maps.a[s][0], c.x.hi, c.x.N, c.x.D, c.x.H, c.x.W, c.x.C, c.x.ld, KC, box ? HaloTile::BW : a.tw,
                          box ? HaloTile::BH : a.th, box ? (pair ? HaloBox<2>::BD : HaloTile::BD) : a.td, estride, swz, c.x.vD,
                          c.x.vH, c.x.vW));
    B200_TRY(make_w_map(&maps.b[s][0], c.w_hi, a.ntaps[s], op.Cop, c.Cip, KC, BN, swz));
    if (split) {
      B200_TRY(make_act_map(&maps.a[s][1], c.x.lo, c.x.N, c.x.D, c.x.H, c.x.W, c.x.C, c.x.ld, KC, a.tw, a.th, a.td,
                            estride, swz, c.x.vD, c.x.vH, c.x.vW));
      B200_TRY(make_w_map(&maps.b[s][1], c.w_lo, a.ntaps[s], op.Cop, c.Cip, KC, BN, swz));
    }
  }
  a.npass = r.npass;
  a.mode = op.mode;
  a.out_hi = out.hi; a.out_lo = out.lo; a.ldo = out.ld;
  ConvClassMaps cmaps;
  memset(&cmaps, 0, sizeof(cmaps));
  if (cls) {
    // data gradient of y[o] = sum_k x[2o + k - 1] w[k]: dx[2j] = dy[j] w[1]; dx[2j+1] = dy[j] w[2] + dy[j+1] w[0].  With the
    // flipped pack Wd[k'] = w[2 - k'] (what emit_dgrad binds): even outputs use k' = 1 (delta 0), odd outputs k' = 0
    // (delta 0) and k' = 2 (delta +1); dy[j+1] beyond the grid reads as zero (TMA out-of-bounds fill).
    // cls_mode 2 (ConvTranspose3d, kernel = stride = 2): out[2j + p] = x[j] w[p], one tap per class
    a.cls_mode = op.cls_mode;
    const int cbo = BN < 64 ? BN : 64;
    for (int c = 0; c < 8; ++c) {
      const int pd = (c >> 2) & 1, ph = (c >> 1) & 1, pw = c & 1;
      int n = 0;
      if (op.cls_mode == 2) a.cls_tap[c][n++] = (unsigned char)c;   // tap index kd*4 + kh*2 + kw = the class itself
      else
      for (int kd = 0; kd < 3; ++kd)
        for (int kh = 0; kh < 3; ++kh)
          for (int kw = 0; kw < 3; ++kw) {
            const bool ok = (pd ? kd != 1 : kd == 1) && (ph ? kh != 1 : kh == 1) && (pw ? kw != 1 : kw == 1);
            if (!ok) continue;
            a.cls_tap[c][n++] = (unsigned char)((kd * 9 + kh * 3 + kw) | ((kw == 2) << 5) | ((kh == 2) << 6) | ((kd == 2) << 7));
          }
      a.cls_n[c] = (unsigned char)n;
      B200_TRY(make_act_map_class(&cmaps.oc[c][0], out.hi, out.N, out.D, out.H, out.W, out.C, out.ld, pd, ph, pw, cbo, a.tw, a.th,
                                  a.td, swz_for_bytes(cbo * 2)));
      if (split)
        B200_TRY(make_act_map_class(&cmaps.oc[c][1], out.lo, out.N, out.D, out.H, out.W, out.C, out.ld, pd, ph, pw, cbo, a.tw,
                                    a.th, a.td, swz_for_bytes(cbo * 2)));
    }
    // single-pass bf16: the two W-parity classes of a (pd, ph) pair share one dense store (see tmap.h); the pair maps replace the
    // even classes' descriptors
    if (r.cls_pair) {
      for (int c = 0; c < 8; c += 2)
        B200_TRY(make_act_map_classpair(&cmaps.oc[c][0], out.hi, out.N, out.D, out.H, out.W, out.C, out.ld, (c >> 2) & 1, (c >> 1) & 1, cbo,
                                        2 * a.tw, a.th, a.td, swz_for_bytes(cbo * 2)));
      a.cls_pair = 1;
    }
    maps.o[0] = cmaps.oc[0][0];   // keeps the (unused) plain output descriptor valid
  } else {
    const int cbo = BN < 64 ? BN : 64;
    const int otd = wide ? a.td / 2 : a.td;   // the 256-voxel tile: each warpgroup stores its half
    B200_TRY(make_act_map(&maps.o[0], out.hi, out.N, out.D, out.H, out.W, out.C, out.ld, cbo, a.tw, a.th, otd, 1,
                          swz_for_bytes(cbo * 2)));
    if (split || out.lo)   // bf16 operands with a lo output: the fp32 accumulators stored as hi + lo (MONAI UNet's logits)
      B200_TRY(make_act_map(&maps.o[1], out.lo, out.N, out.D, out.H, out.W, out.C, out.ld, cbo, a.tw, a.th, otd, 1,
                            swz_for_bytes(cbo * 2)));
  }
  if (op.res) {
    a.res_hi = op.res->hi; a.res_lo = op.res->lo; a.ldr = op.res->ld;
  }
  a.scale = op.scale;
  a.bias = op.bias; a.zero_last = op.zero_last;
  a.stats = op.stats; a.stats_ld = op.stats_ld;
  if (op.mode == 1) {
    a.x_hi = op.gn_x->hi; a.x_lo = op.gn_x->lo; a.ldx = op.gn_x->ld;
    a.coef = reinterpret_cast<const float4*>(op.coef); a.coef_ld = op.coef_ld;
    a.slope = op.slope; a.bstats = op.bstats;
  }
  const dim3 grid((unsigned)r.grid[0], (unsigned)r.grid[1], (unsigned)r.grid[2]);
  return with_conv_kernel(r.kind, BN, KC, r.wgs, [&](auto k) {
    return launch_cfg<decltype(k)::BN, decltype(k)::KC, decltype(k)::MODE>(maps, a, grid, st, cmaps);
  });
}

}  // namespace b200
