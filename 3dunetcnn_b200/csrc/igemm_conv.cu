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
#include <cstdlib>
#include <type_traits>
#include "conv_common.cuh"

namespace b200 {

// Kernel modes: per-tap streaming tiles, class mode (parity-class data gradient / k = s = 2 transposed convolution), and halo
// mode: the 3x3x3 stride-1 source is loaded as ONE halo box (KC, 10, 18, 3) per K chunk for an 8 x 16 x 1 output tile, and the
// 27 taps read it through shifted shared-memory descriptors (27x less activation traffic from L2 than per-tap boxes).
// CONV_HALO_WS is halo mode on the persistent, weight-stationary kernel (k_igemm_conv_halo_ws) for the (BN, KC) whose 27 weight
// tiles fit in shared memory beside the halo box; CONV_HALO runs the ring kernel below for the wider ones.
enum ConvMode { CONV_STREAM = 0, CONV_CLASS = 1, CONV_HALO = 2, CONV_HALO_WS = 3 };

// Shared memory: STAGES-deep TMA ring | fp32 accumulator tile [128][BN + 4] | (class mode) output staging | (halo mode) halo box
// | aux.  Outside class mode the output staging tile reuses the ring: the CTA computes one tile, so every stage has been consumed
// when the epilogue starts.  Class mode keeps the staging tile apart because the producer is already loading the next class.
// BN <= 32 (<= 204 registers per thread) sizes the ring so that two CTAs share an SM (one CTA's epilogue overlaps the other's
// MMAs) when that still leaves four stages; otherwise one CTA takes up to 227 KB.
template <int BN, int KC, int MODE>
struct ConvCfg {
  static constexpr int A_BYTES = 128 * KC * 2;
  static constexpr int B_BOX_BYTES = BN * KC * 2;
  static constexpr int B_BYTES = B_BOX_BYTES < 1024 ? 1024 : B_BOX_BYTES;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int ACC_LD = BN + 4;                     // floats per accumulator row: 16-byte aligned, rows on staggered banks
  static constexpr int ACC_BYTES = 128 * ACC_LD * 4;
  static constexpr int AUX_BYTES = 1024 + 4 * BN * 2 * 4 + BN * 16;  // barriers | per-warp stats | coef
  static constexpr int OUT_STAGING = 2 * 128 * BN * 2;    // hi + lo output tiles (class pairs: 256 rows of hi)
  static constexpr int STG_BYTES = MODE == CONV_CLASS ? OUT_STAGING : 0;
  static constexpr int RB = KC * 2;                        // bytes per voxel row of an activation tile
  static constexpr int HALO_TX = 540 * RB;                 // 10 x 18 x 3 voxels
  static constexpr int HALO_BYTES = MODE == CONV_HALO ? (HALO_TX + 1023) / 1024 * 1024 : 0;
  static constexpr int FIXED = ACC_BYTES + STG_BYTES + HALO_BYTES + AUX_BYTES + 1024;   // +1024 alignment slack
  static constexpr int SMEM_LIMIT = 232448;                // sm_90 opt-in dynamic shared memory per block
  static constexpr int TWO_PER_SM = 115712;                // 228 KB per SM, 1 KB reserved per block
  static constexpr int MIN_BLOCKS = BN <= 32 ? 2 : 1;      // 2 x 160 threads x <= 204 registers fit the 64 K register file
  static constexpr int STAGES_2 = MIN_BLOCKS == 2 ? (TWO_PER_SM - FIXED) / STAGE_BYTES : 0;
  static constexpr int STAGES_RAW = STAGES_2 >= 4 ? STAGES_2 : (SMEM_LIMIT - FIXED) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 6 ? 6 : STAGES_RAW;
  static constexpr int BLOCKS_PER_SM = STAGES_2 >= 4 ? 2 : 1;
  static constexpr int PIPE_BYTES = STAGES * STAGE_BYTES > OUT_STAGING ? STAGES * STAGE_BYTES : OUT_STAGING;
  static constexpr int SMEM_BYTES = PIPE_BYTES + FIXED;
  static constexpr uint32_t LAYOUT = swizzle_for_row_bytes(KC * 2);
  static constexpr uint32_t SBO = 8 * KC * 2;
  static_assert(STAGES >= 2 && SMEM_BYTES <= SMEM_LIMIT, "igemm_conv: configuration does not fit shared memory");
};

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
  float* s_acc = reinterpret_cast<float*>(smem + Cfg::PIPE_BYTES);
  uint8_t* stage_out = MODE == CONV_CLASS ? smem + Cfg::PIPE_BYTES + Cfg::ACC_BYTES : smem;
  uint8_t* halo = smem + Cfg::PIPE_BYTES + Cfg::ACC_BYTES + Cfg::STG_BYTES;
  uint8_t* aux = halo + Cfg::HALO_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(aux);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;
  uint64_t* halo_full = empty_bar + Cfg::STAGES;
  uint64_t* halo_empty = halo_full + 1;
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
    mbar_init(halo_empty, 4);
    fence_barrier_init();
  }
  pdl_wait();   // before the first global read (the coefficient table below); the barrier set-up above overlaps the previous kernel
  if (warp < 4) {
    const int e = threadIdx.x;
    for (int i = e; i < 4 * BN * 2; i += 128) s_stats[i] = 0.f;
    if (p.mode == 1) {
      for (int c = e; c < BN; c += 128)
        s_coef[c] = (n0 + c < p.Cout) ? p.coef[(long long)n * p.coef_ld + n0 + c] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  __syncthreads();
  pdl_launch_dependents();

  // class mode: ONE CTA computes all eight parity classes of its voxel tile (27 tap products walked class by class, each class
  // drained by the epilogue before the next one starts).  One CTA per class would spend most of its life in set-up.
  int total_iters = (p.ntaps[0] * p.kchunks[0] + p.ntaps[1] * p.kchunks[1]) * p.npass;
  if (p.cls_mode) {
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
        // one halo box per K chunk (its zero padding = TMA out-of-bounds fill), then the 27 taps' weight tiles
        for (int kc = 0; kc < p.kchunks[0]; ++kc) {
          mbar_wait(halo_empty, (kc & 1) ^ 1);
          mbar_expect_tx_if(issue, halo_full, Cfg::HALO_TX);
          tma_load_5d_if(issue, halo, &maps.a[0][0], halo_full, kc * KC, w0 - 1, h0 - 1, d0 - 1, n);
          for (int tap = 0; tap < 27; ++tap) {
            const int s = it % Cfg::STAGES;
            mbar_wait(&empty_bar[s], ((it / Cfg::STAGES) & 1) ^ 1);
            mbar_expect_tx_if(issue, &full_bar[s], Cfg::B_BOX_BYTES);
            tma_load_3d_if(issue, smem + s * Cfg::STAGE_BYTES + Cfg::A_BYTES, &maps.b[0][0], &full_bar[s], kc * KC, n0, tap);
            ++it;
          }
        }
        continue;
      }
      for (int cls = 0; cls < (p.cls_mode ? 8 : 1); ++cls) {
        const int ntap_loop = p.cls_mode ? (int)p.cls_n[cls] : nt;
        for (int ti = 0; ti < ntap_loop; ++ti) {
          int tap = ti, cw, ch, cd;
          if (p.cls_mode) {   // class tap list: source voxel j + delta, packed-weight tap index
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
              uint8_t* sa = smem + s * Cfg::STAGE_BYTES;
              tma_load_5d_if(issue, sa, &maps.a[src][pass == 1], &full_bar[s], kc * KC, cw, ch, cd, n);
              tma_load_3d_if(issue, sa + Cfg::A_BYTES, &maps.b[src][pass == 2], &full_bar[s], kc * KC, n0, tap);
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
    return p.cls_mode
        ? (((long long)n * (2 * p.Do) + 2 * d + ((cls >> 2) & 1)) * (2 * p.Ho) + 2 * h + ((cls >> 1) & 1)) * (2 * p.Wo) + 2 * w + (cls & 1)
        : (((long long)n * p.Do + d) * p.Ho + h) * p.Wo + w;
  };
  for (int cls = 0; cls < (p.cls_mode ? 8 : 1); ++cls) conv_epilogue_prefetch(p, n0, BN, vox_of(cls), valid);   // -> L2 while the MMAs run

  float acc[2][BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
  // halo mode: the halo box holds rows ((dz * 18) + hy) * 10 + wx; output row r = h * 8 + w of tap (kd, kh, kw) reads halo row
  // (kd * 18 + h + kh) * 10 + w + kw, so each 8-row group (one h) is 8 consecutive halo rows and the next group starts one halo
  // row of 10 voxels further (SBO).  The descriptors start at arbitrary row offsets inside the swizzled box: the swizzle is a
  // function of the absolute shared-memory address, for the TMA writes and for the wgmma reads alike.
  constexpr uint32_t hi_halo = desc_hi(10 * Cfg::RB, Cfg::LAYOUT);
  const uint32_t halo_lo0 = desc_lo(smem_u32(halo), 16);
  const int halo_iters = MODE == CONV_HALO ? 27 * p.kchunks[0] : 0;
  int it = 0;
  for (int cls = 0; cls < (p.cls_mode ? 8 : 1); ++cls) {
    const int n_it = p.cls_mode ? (int)p.cls_n[cls] * p.kchunks[0] * p.npass : total_iters;
    int prev = -1;   // ring slot whose MMAs may still be reading it
    for (int i = 0; i < n_it; ++i, ++it) {
      const int s = it % Cfg::STAGES;
      const bool from_halo = i < halo_iters;
      const int tap = i % 27;
      if (from_halo && tap == 0) mbar_wait(halo_full, (i / 27) & 1);
      mbar_wait(&full_bar[s], (it / Cfg::STAGES) & 1);
      uint32_t a_lo = desc_lo(smem0 + s * Cfg::STAGE_BYTES, 16), a_hi = hi_d, a_half = HALF_M;
      if (MODE == CONV_HALO && from_halo) {
        const int kd = tap / 9, kh = (tap / 3) % 3, kw = tap % 3;
        a_lo = halo_lo0 + (((kd * 180 + kh * 10 + kw) * Cfg::RB) >> 4);
        a_hi = hi_halo;
        a_half = (80 * Cfg::RB) >> 4;   // rows 64-127 = h 8..15
      }
      const uint32_t b_lo = desc_lo(smem0 + s * Cfg::STAGE_BYTES + Cfg::A_BYTES, 16);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < KC / 16; ++k) {
        const uint32_t accumulate = (i > 0 || k > 0) ? 1u : 0u;   // the first K step of a class overwrites the accumulator
        Wgmma<BN>::template mma<0, 0>(acc[0], desc_from(a_lo + 2 * k, a_hi), desc_from(b_lo + 2 * k, hi_d), accumulate);
        Wgmma<BN>::template mma<0, 0>(acc[1], desc_from(a_lo + a_half + 2 * k, a_hi), desc_from(b_lo + 2 * k, hi_d), accumulate);
      }
      wgmma_commit();
      if (from_halo && tap == 26) {
        // last tap of a halo box: the producer can load the next chunk's box only once every MMA reading this one is done,
        // and the next MMA needs that box -- so drain here instead of deferring the hand-back by one stage
        wgmma_wait<0>();
        if (lane == 0) {
          if (prev >= 0) mbar_arrive(&empty_bar[prev]);
          mbar_arrive(&empty_bar[s]);
          mbar_arrive(halo_empty);
        }
        prev = -1;
      } else {
        wgmma_wait<1>();   // the previous stage's MMAs are complete: hand its slot back to the producer
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = s;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc[0]);
    wgmma_fence_regs(acc[1]);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);

    // accumulator fragments -> s_acc (row-major), so that each thread drains one output voxel row below
    const bool pair = p.cls_pair != 0, pair_first = pair && (cls & 1) == 0, pair_second = pair && (cls & 1) == 1;
    if (cls > 0) {
      if (!pair_second && threadIdx.x == 0) tma_store_wait_read0();    // the previous stores have read the staging tile
      asm volatile("bar.sync 1, 128;" ::: "memory");                   // and every thread has read its s_acc row
    }
#pragma unroll
    for (int hm = 0; hm < 2; ++hm) {
      const int r0 = hm * 64 + warp * 16 + (lane >> 2);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = j * 8 + 2 * (lane & 3);
        *reinterpret_cast<float2*>(s_acc + r0 * Cfg::ACC_LD + c) = make_float2(acc[hm][4 * j], acc[hm][4 * j + 1]);
        *reinterpret_cast<float2*>(s_acc + (r0 + 8) * Cfg::ACC_LD + c) = make_float2(acc[hm][4 * j + 2], acc[hm][4 * j + 3]);
      }
    }
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
        const CUtensorMap* mo_hi = p.cls_mode ? &cmaps.oc[cls][0] : &maps.o[0];
        const CUtensorMap* mo_lo = p.cls_mode ? &cmaps.oc[cls][1] : &maps.o[1];
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
    double* dst = (p.mode == 0) ? p.stats : p.bstats;
    const int ld = (p.mode == 0) ? p.stats_ld : p.coef_ld;
    for (int c = threadIdx.x; c < BN * 2; c += 128) {
      const float v = s_stats[c] + s_stats[BN * 2 + c] + s_stats[2 * BN * 2 + c] + s_stats[3 * BN * 2 + c];
      if (n0 + (c >> 1) < p.Cout) atomicAdd(&dst[((long long)n * ld + n0) * 2 + c], (double)v);
    }
  }
  if (threadIdx.x == 0) tma_store_wait_all();   // the staging tile must outlive the bulk store
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
struct HaloWsCfg {
  static constexpr int A_BYTES = 128 * KC * 2;
  static constexpr int B_BOX_BYTES = BN * KC * 2;
  static constexpr int B_BYTES = B_BOX_BYTES < 1024 ? 1024 : B_BOX_BYTES;
  static constexpr int STAGES = 2;                          // second-source ring
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int ACC_LD = BN + 4;
  static constexpr int ACC_BYTES = 128 * ACC_LD * 4;        // > the 128 x BN bf16 staging tile
  static constexpr int W_BYTES = (27 * B_BOX_BYTES + 1023) / 1024 * 1024;
  static constexpr int R_RAW = STAGES * STAGE_BYTES > ACC_BYTES ? STAGES * STAGE_BYTES : ACC_BYTES;
  static constexpr int R_BYTES = (R_RAW + 1023) / 1024 * 1024;
  static constexpr int RB = KC * 2;
  static constexpr int HALO_TX = 540 * RB;
  static constexpr int HALO_BYTES = (HALO_TX + 1023) / 1024 * 1024;
  static constexpr int AUX_BYTES = 1024 + 4 * BN * 2 * 4 + BN * 16;   // barriers | per-warp stats | coef
  static constexpr int FIXED = W_BYTES + R_BYTES + AUX_BYTES + 1024;  // +1024 alignment slack
  static constexpr int BLOCKS_PER_SM = BN <= 32 ? 2 : 1;
  static constexpr int BUDGET = BLOCKS_PER_SM == 2 ? ConvCfg<BN, KC, CONV_STREAM>::TWO_PER_SM : ConvCfg<BN, KC, CONV_STREAM>::SMEM_LIMIT;
  static constexpr int HALO_BUFS = FIXED + 2 * HALO_BYTES <= BUDGET ? 2 : 1;
  static constexpr int SMEM_BYTES = FIXED + HALO_BUFS * HALO_BYTES;
  // BN <= 64: the accumulator row a thread holds in registers during the epilogue stays at <= 64 floats
  static constexpr bool FITS = BN <= 64 && SMEM_BYTES <= BUDGET;
  static constexpr uint32_t LAYOUT = swizzle_for_row_bytes(KC * 2);
  static constexpr uint32_t SBO = 8 * KC * 2;
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
  uint8_t* aux = halo + Cfg::HALO_BUFS * Cfg::HALO_BYTES;
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
    w0 = (t % p.tiles_w) * 8; t /= p.tiles_w;
    h0 = (t % p.tiles_h) * 16; t /= p.tiles_h;
    d0 = t % p.tiles_d;
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
      tma_load_5d_if(issue, halo + hb * Cfg::HALO_BYTES, &maps.a[0][0], &halo_full[hb], 0, w0 - 1, h0 - 1, d0 - 1, n);
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
  constexpr uint32_t hi_halo = desc_hi(10 * Cfg::RB, Cfg::LAYOUT);   // see k_igemm_conv: 8-row groups are 10 halo rows apart
  constexpr uint32_t HALF_M = (64 * KC * 2) >> 4;                    // ring A tile: row 64
  constexpr uint32_t HALO_HALF = (80 * Cfg::RB) >> 4;                // halo: output rows 64-127 = h 8..15
  const uint32_t w_lo0 = desc_lo(smem_u32(wts), 16);
  const uint32_t halo_lo0 = desc_lo(smem_u32(halo), 16);
  const uint32_t reg0 = smem_u32(reg);
  const int row = threadIdx.x;
  const int wl = row % 8, hl = row / 8;
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
    const uint32_t hlo = halo_lo0 + ((hb * Cfg::HALO_BYTES) >> 4);
    float acc[2][BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    mbar_wait(&halo_full[hb], (j / Cfg::HALO_BUFS) & 1);
    wgmma_fence();
#pragma unroll
    for (int tap = 0; tap < 27; ++tap) {
      const int kd = tap / 9, kh = (tap / 3) % 3, kw = tap % 3;
      const uint32_t a_lo = hlo + (((kd * 180 + kh * 10 + kw) * Cfg::RB) >> 4);
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
      for (int c = threadIdx.x; c < BN; c += 128)
        s_coef[c] = (n0 + c < p.Cout) ? p.coef[(long long)n * p.coef_ld + n0 + c] : make_float4(0.f, 0.f, 0.f, 0.f);
      coef_n = n;
    }
#pragma unroll
    for (int hm = 0; hm < 2; ++hm) {
      const int r0 = hm * 64 + warp * 16 + (lane >> 2);
#pragma unroll
      for (int jj = 0; jj < BN / 8; ++jj) {
        const int c = jj * 8 + 2 * (lane & 3);
        *reinterpret_cast<float2*>(s_acc + r0 * Cfg::ACC_LD + c) = make_float2(acc[hm][4 * jj], acc[hm][4 * jj + 1]);
        *reinterpret_cast<float2*>(s_acc + (r0 + 8) * Cfg::ACC_LD + c) = make_float2(acc[hm][4 * jj + 2], acc[hm][4 * jj + 3]);
      }
    }
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
    if (want_stats) {   // this tile's fp32 partials -> one fp64 atomic per channel; the slots restart from zero
      for (int c = threadIdx.x; c < BN * 2; c += 128) {
        const float v = s_stats[c] + s_stats[BN * 2 + c] + s_stats[2 * BN * 2 + c] + s_stats[3 * BN * 2 + c];
        s_stats[c] = 0.f; s_stats[BN * 2 + c] = 0.f; s_stats[2 * BN * 2 + c] = 0.f; s_stats[3 * BN * 2 + c] = 0.f;
        if (n0 + (c >> 1) < p.Cout) atomicAdd(&stats_dst[((long long)n * stats_ld + n0) * 2 + c], (double)v);
      }
    }
  }
  if (threadIdx.x == 0) tma_store_wait_all();   // the staging tile must outlive the bulk store
}

// ----------------------------------------------------------------------------------------------- host side
static void pick_tile(int Wo, int Ho, int Do, int& tw, int& th, int& td) {
  tw = Wo >= 8 ? 8 : Wo >= 4 ? 4 : Wo >= 2 ? 2 : 1;
  int rem = 128 / tw;
  th = Ho >= 4 ? 4 : Ho >= 2 ? 2 : 1;
  if (th > rem) th = rem;
  td = rem / th;
}

// The compile-time configuration of the kernel a (BN, KC, MODE) launch runs.
template <int BN, int KC, int MODE>
using ConvCfgOf = std::conditional_t<MODE == CONV_HALO_WS, HaloWsCfg<BN, KC>, ConvCfg<BN, KC, MODE>>;

template <int BN, int KC, int MODE>
static int launch_cfg(const ConvMaps& maps, const ConvArgs& args, dim3 grid, cudaStream_t st, const ConvClassMaps& cmaps) {
  using Cfg = ConvCfgOf<BN, KC, MODE>;
  static bool attr_set[64] = {false};
  int dev = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  if (dev < 64 && !attr_set[dev]) {
    if constexpr (MODE == CONV_HALO_WS)
      B200_CHECK_CUDA(cudaFuncSetAttribute(k_igemm_conv_halo_ws<BN, KC>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    else
      B200_CHECK_CUDA(cudaFuncSetAttribute(k_igemm_conv<BN, KC, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set[dev] = true;
  }
  if constexpr (MODE == CONV_HALO_WS)
    launch_pdl(k_igemm_conv_halo_ws<BN, KC>, grid, dim3(160), Cfg::SMEM_BYTES, st, maps, args);
  else
    launch_pdl(k_igemm_conv<BN, KC, MODE>, grid, dim3(160), Cfg::SMEM_BYTES, st, maps, args, cmaps);
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
  const int c = op.src[k].x.C;
  return c > 32 ? 64 : c > 16 ? 32 : 16;
}

static int conv_bn(const ConvOp& op) {
  const int BN = op.out.C > 64 ? 128 : op.out.C > 32 ? 64 : op.out.C > 16 ? 32 : 16;
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

// Halo mode (see ConvMode) for 3x3x3 stride-1 convolutions (plus an optional fused 1x1x1 source) whose output planes fill the
// 8 x 16 tile, in single-pass bf16, when it keeps the configuration's CTAs per SM.  Inputs wider than 64 channels take several
// halo boxes per tile, drained one after the other;
// they stay on per-tap tiles unless voxels * Cout >= B200UNET_HALO_WIDE_MIN (tests set it to 0 to reach that path with
// oracle-sized shapes; off by default: the forward category of the C2 step was slower with them in halo mode on the H100).  B200UNET_NO_HALO=1 keeps every launch on the per-tap kernel (A/B measurements).
bool conv_halo_eligible(const ConvOp& op) {
  static const bool off = getenv("B200UNET_NO_HALO") && atoi(getenv("B200UNET_NO_HALO")) != 0;
  if (off || op.cls_mode) return false;
  const ConvSrc& c = op.src[0];
  if (c.ksz != 3 || c.stride != 1 || c.nopad) return false;
  if (op.nsrc == 2 && (op.src[1].ksz != 1 || op.src[1].stride != 1)) return false;
  for (int s = 0; s < op.nsrc; ++s)
    if (op.src[s].x.lo || op.src[s].w_lo) return false;
  long long wide_min = -1;
  if (const char* e = getenv("B200UNET_HALO_WIDE_MIN")) wide_min = atoll(e);
  if (c.x.C > 64 && (wide_min < 0 || (long long)op.out.N * op.out.D * op.out.H * op.out.W * op.out.C < wide_min)) return false;
  return op.out.W >= 8 && op.out.H >= 16 && halo_keeps_occupancy(conv_bn(op), conv_kc(op));
}

template <int BN_, int KC_, int MODE_>
struct ConvKernel { static constexpr int BN = BN_, KC = KC_, MODE = MODE_; };

// f(ConvKernel<BN, KC, MODE>{}) for the instantiated kernel of (kind, BN, KC): the one selection conv_route reports and
// launch_igemm_conv launches.  E_UNSUPPORTED when no such kernel is instantiated.
template <class F>
static int with_conv_kernel(int kind, int BN, int KC, F&& f) {
#define B200_CONV_CASE(bn, kc)                                                                              \
  if (BN == bn && KC == kc) {                                                                               \
    if (kind == CONV_KIND_CLASS1 || kind == CONV_KIND_CLASS2) {                                             \
      if constexpr (bn <= 64) return f(ConvKernel<bn, kc, CONV_CLASS>{});                                   \
    } else if (kind == CONV_KIND_HALO) {                                                                    \
      if constexpr (halo_keeps_occupancy<bn, kc>()) return f(ConvKernel<bn, kc, halo_mode<bn, kc>()>{});    \
    } else {                                                                                                \
      return f(ConvKernel<bn, kc, CONV_STREAM>{});                                                          \
    }                                                                                                       \
  }
  B200_CONV_CONFIGS(B200_CONV_CASE)
#undef B200_CONV_CASE
  set_error("igemm_conv: no kernel for BN=%d KC=%d (kind %d)", BN, KC, kind);
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
  const bool halo = conv_halo_eligible(op);
  r->kind = op.cls_mode == 1 ? CONV_KIND_CLASS1 : op.cls_mode == 2 ? CONV_KIND_CLASS2 : halo ? CONV_KIND_HALO : CONV_KIND_TAP;
  if (halo) {   // 8 x 16 output plane tiles
    r->tw = 8; r->th = 16; r->td = 1;
  } else {
    pick_tile(gW, gH, gD, r->tw, r->th, r->td);
  }
  r->tiles_w = ceil_div(gW, r->tw); r->tiles_h = ceil_div(gH, r->th); r->tiles_d = ceil_div(gD, r->td);
  r->KC = conv_kc(op);
  r->BN = conv_bn(op);
  for (int s = 0; s < op.nsrc; ++s) r->kchunks[s] = ceil_div(op.src[s].x.C, r->KC);
  r->npass = split ? 3 : 1;
  r->cls_pair = op.cls_mode && !split ? 1 : 0;
  r->grid[0] = (int)((long long)out.N * r->tiles_d * r->tiles_h * r->tiles_w);
  r->grid[1] = ceil_div(out.C, r->BN);
  r->grid[2] = 1;
  return with_conv_kernel(r->kind, r->BN, r->KC, [&](auto k) {
    using Cfg = ConvCfgOf<decltype(k)::BN, decltype(k)::KC, decltype(k)::MODE>;
    r->stages = Cfg::STAGES; r->blocks_per_sm = Cfg::BLOCKS_PER_SM; r->smem_bytes = Cfg::SMEM_BYTES;
    if constexpr (decltype(k)::MODE == CONV_HALO_WS) {
      // persistent CTAs: one wave (max_ctas, a diagnostics cap, makes small shapes walk several tiles per CTA)
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
  const bool split = r.npass == 3, halo = r.kind == CONV_KIND_HALO, cls = op.cls_mode != 0;
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
    B200_TRY(make_act_map(&maps.a[s][0], c.x.hi, c.x.N, c.x.D, c.x.H, c.x.W, c.x.C, c.x.ld, KC, a.tw, a.th, a.td,
                          estride, swz, c.x.vD, c.x.vH, c.x.vW));
    B200_TRY(make_w_map(&maps.b[s][0], c.w_hi, a.ntaps[s], op.Cop, c.Cip, KC, BN, swz));
    if (split) {
      B200_TRY(make_act_map(&maps.a[s][1], c.x.lo, c.x.N, c.x.D, c.x.H, c.x.W, c.x.C, c.x.ld, KC, a.tw, a.th, a.td,
                            estride, swz, c.x.vD, c.x.vH, c.x.vW));
      B200_TRY(make_w_map(&maps.b[s][1], c.w_lo, a.ntaps[s], op.Cop, c.Cip, KC, BN, swz));
    }
  }
  if (halo) {
    const ConvSrc& c = op.src[0];
    B200_TRY(make_act_map(&maps.a[0][0], c.x.hi, c.x.N, c.x.D, c.x.H, c.x.W, c.x.C, c.x.ld, KC, 10, 18, 3, 1, swz, c.x.vD, c.x.vH,
                          c.x.vW));
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
    B200_TRY(make_act_map(&maps.o[0], out.hi, out.N, out.D, out.H, out.W, out.C, out.ld, cbo, a.tw, a.th, a.td, 1,
                          swz_for_bytes(cbo * 2)));
    if (split)
      B200_TRY(make_act_map(&maps.o[1], out.lo, out.N, out.D, out.H, out.W, out.C, out.ld, cbo, a.tw, a.th, a.td, 1,
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
  return with_conv_kernel(r.kind, BN, KC, [&](auto k) {
    return launch_cfg<decltype(k)::BN, decltype(k)::KC, decltype(k)::MODE>(maps, a, grid, st, cmaps);
  });
}

}  // namespace b200
