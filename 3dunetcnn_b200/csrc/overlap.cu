// Overlap counts of segmentations (MONAI DiceMetric, MeanIoU, ConfusionMatrixMetric): one pass over a batch of predictions and
// targets that counts, for every (item b, class c), P = voxels predicted as c, G = voxels whose target is c and I = voxels that are
// both.  Every metric of those classes is a few operations on (P, G, I) and the voxel count S.
//
// Each operand is in one of these forms (OverlapForm):
//   one-hot      [B][C][S] uint8 (bool) or fp32: class c iff the value is nonzero
//   label map    [B][1][S] uint8 or int64: the class is the value; a value outside [0, C) is no class
//   threshold    [B][C][S] fp32 scores: class c iff x >= thr (the caller turns "sigmoid(x) > 0.5" into one compare)
//   argmax       [B][C][S] fp32 scores: the class is the first channel of the largest score (torch.argmax: NaN is largest)
// The target takes the first two.  The prediction takes all four.
//
// grid (X, B): block (x, b) walks the tiles x, x + X, ... of item b.  A tile holds kTile voxels; thread t owns voxels
// t + k kThreads (k < kVPT) of it, so every warp load reads consecutive voxels of one channel.
//   label map / argmax operands: each owned voxel's class is kept in a register.
//   both operands single-class: the (pred, target) class pairs of a warp are grouped with match.any and one lane per group
//                    adds the group's size to the block's counters (shared-memory atomics).
//   otherwise:       for each class c, every thread counts (p, g, p & g) over its voxels, packed in one word (fields <= kVPT,
//                    so a warp total < 256 per field), adds them across the warp with redux.sync, and lane 0 adds them to the
//                    block's counters.
// The block's 32-bit counters (at most S < 2^31 each) are added once to the int64 counts [B][C][3] with integer atomics, after
// a memset that is part of the call: exact, and the same whatever order the blocks run in.  No host synchronisation.
#include "kernels.h"

namespace b200 {
namespace {

constexpr int kThreads = 256;
constexpr int kVPT = 4;                     // voxels per thread per tile
constexpr int kTile = kThreads * kVPT;
constexpr int kSMs = 132;                   // H100 SXM; with 8 blocks per SM it sets the grid from the shape alone
constexpr int kBlocksPerSM = 2048 / kThreads;

template <int F>
__host__ __device__ constexpr bool single_class() { return F == OV_LABEL_U8 || F == OV_LABEL_I64 || F == OV_ARGMAX_F32; }

// the classes of voxels s0 + k kThreads (k < kVPT) of item b (label map, argmax), -1 for none or past S.  Argmax walks the channels
// once for all kVPT voxels, so each step has kVPT independent loads in flight.
template <int F>
__device__ __forceinline__ void classes_of(const OverlapOperand& o, int b, int C, long long S, long long s0, int (&cls)[kVPT]) {
  if (F == OV_LABEL_U8 || F == OV_LABEL_I64) {
#pragma unroll
    for (int k = 0; k < kVPT; ++k) {
      const long long s = s0 + k * kThreads;
      long long l = -1;
      if (s < S)
        l = F == OV_LABEL_U8 ? (long long)__ldg(static_cast<const uint8_t*>(o.data) + (long long)b * S + s)
                             : __ldg(static_cast<const long long*>(o.data) + (long long)b * S + s);
      cls[k] = l >= 0 && l < C ? (int)l : -1;
    }
  } else {
    const float* x = static_cast<const float*>(o.data) + (long long)b * C * S + s0;
    float best[kVPT];
#pragma unroll
    for (int k = 0; k < kVPT; ++k) {
      best[k] = s0 + k * kThreads < S ? __ldg(x + k * kThreads) : 0.f;
      cls[k] = s0 + k * kThreads < S ? 0 : -1;
    }
    for (int c = 1; c < C; ++c) {
#pragma unroll
      for (int k = 0; k < kVPT; ++k) {
        const float v = s0 + k * kThreads < S ? __ldg(x + (long long)c * S + k * kThreads) : 0.f;
        // strictly larger, or the first NaN; ties keep the lower index
        if (best[k] == best[k] && !(v <= best[k])) { best[k] = v; cls[k] = c; }
      }
    }
    if (s0 + (kVPT - 1) * kThreads >= S)
#pragma unroll
      for (int k = 0; k < kVPT; ++k)
        if (s0 + k * kThreads >= S) cls[k] = -1;
  }
}

// is voxel s of item b in class c (one-hot, threshold)
template <int F>
__device__ __forceinline__ unsigned in_class(const OverlapOperand& o, int b, int c, int C, long long S, long long s) {
  const long long e = ((long long)b * C + c) * S + s;
  if (F == OV_ONEHOT_U8) return __ldg(static_cast<const uint8_t*>(o.data) + e) != 0;
  if (F == OV_ONEHOT_F32) return __ldg(static_cast<const float*>(o.data) + e) != 0.f;
  return __ldg(static_cast<const float*>(o.data) + e) >= o.thr;
}

template <int PF, int GF>
__global__ void __launch_bounds__(kThreads) k_overlap_counts(OverlapOperand pred, OverlapOperand gt, int C, long long S,
                                                             unsigned long long* __restrict__ counts) {
  __shared__ unsigned cnt[3][B200_OVERLAP_MAX_CLASSES];   // P, G, I of this block
  for (int i = threadIdx.x; i < 3 * B200_OVERLAP_MAX_CLASSES; i += kThreads) (&cnt[0][0])[i] = 0;
  __syncthreads();
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const long long tiles = (S + kTile - 1) / kTile;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long s0 = tile * kTile + threadIdx.x;
    int pl[kVPT], gl[kVPT];
    if (single_class<PF>()) classes_of<PF>(pred, b, C, S, s0, pl);
    if (single_class<GF>()) classes_of<GF>(gt, b, C, S, s0, gl);
    if (single_class<PF>() && single_class<GF>()) {
#pragma unroll
      for (int k = 0; k < kVPT; ++k) {
        const int key = (pl[k] + 1) << 8 | (gl[k] + 1);
        const unsigned peers = __match_any_sync(0xffffffffu, key);
        if (key != 0 && lane == __ffs(peers) - 1) {
          const unsigned n = __popc(peers);
          if (pl[k] >= 0) atomicAdd(&cnt[0][pl[k]], n);
          if (gl[k] >= 0) atomicAdd(&cnt[1][gl[k]], n);
          if (pl[k] >= 0 && pl[k] == gl[k]) atomicAdd(&cnt[2][pl[k]], n);
        }
      }
    } else {
#pragma unroll 2
      for (int c = 0; c < C; ++c) {
        unsigned packed = 0;
#pragma unroll
        for (int k = 0; k < kVPT; ++k) {
          const long long s = s0 + k * kThreads;
          if (s < S) {
            const unsigned p = single_class<PF>() ? pl[k] == c : in_class<PF>(pred, b, c, C, S, s);
            const unsigned g = single_class<GF>() ? gl[k] == c : in_class<GF>(gt, b, c, C, S, s);
            packed += p | g << 8 | (p & g) << 16;
          }
        }
        packed = __reduce_add_sync(0xffffffffu, packed);
        if (lane == 0 && packed) {
          atomicAdd(&cnt[0][c], packed & 0xffu);
          atomicAdd(&cnt[1][c], packed >> 8 & 0xffu);
          atomicAdd(&cnt[2][c], packed >> 16);
        }
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * C; i += kThreads) {
    const int c = i / 3, j = i % 3;
    if (cnt[j][c]) atomicAdd(counts + ((long long)b * C + c) * 3 + j, (unsigned long long)cnt[j][c]);
  }
}

// the form of an operand descriptor, or -1 for a kind / dtype pair no kernel reads
int form_of(const OverlapOperand& o) {
  if (o.kind < 0 || o.kind > OV_KIND_ARGMAX || o.dtype < 0 || o.dtype > OV_DTYPE_F32) return -1;
  switch (o.kind * 3 + o.dtype) {
    case OV_KIND_ONEHOT * 3 + OV_DTYPE_U8: return OV_ONEHOT_U8;
    case OV_KIND_ONEHOT * 3 + OV_DTYPE_F32: return OV_ONEHOT_F32;
    case OV_KIND_LABEL * 3 + OV_DTYPE_U8: return OV_LABEL_U8;
    case OV_KIND_LABEL * 3 + OV_DTYPE_I64: return OV_LABEL_I64;
    case OV_KIND_THRESHOLD * 3 + OV_DTYPE_F32: return OV_THRESH_F32;
    case OV_KIND_ARGMAX * 3 + OV_DTYPE_F32: return OV_ARGMAX_F32;
    default: return -1;
  }
}

template <int PF, int GF>
void launch(const OverlapOperand& p, const OverlapOperand& g, int B, int C, long long S, unsigned long long* counts, cudaStream_t st) {
  const long long tiles = (S + kTile - 1) / kTile;
  long long x = ((long long)kSMs * kBlocksPerSM + B - 1) / B;
  if (x > tiles) x = tiles;
  k_overlap_counts<PF, GF><<<dim3((unsigned)x, B), kThreads, 0, st>>>(p, g, C, S, counts);
}

template <int PF>
void launch_gt(int gf, const OverlapOperand& p, const OverlapOperand& g, int B, int C, long long S, unsigned long long* counts,
               cudaStream_t st) {
  switch (gf) {
    case OV_ONEHOT_U8: launch<PF, OV_ONEHOT_U8>(p, g, B, C, S, counts, st); break;
    case OV_ONEHOT_F32: launch<PF, OV_ONEHOT_F32>(p, g, B, C, S, counts, st); break;
    case OV_LABEL_U8: launch<PF, OV_LABEL_U8>(p, g, B, C, S, counts, st); break;
    default: launch<PF, OV_LABEL_I64>(p, g, B, C, S, counts, st); break;
  }
}

}  // namespace

int launch_overlap_counts(const OverlapOperand& pred, const OverlapOperand& gt, int B, int C, int D, int H, int W, int64_t* counts,
                          cudaStream_t st) {
  const int pf = form_of(pred), gf = form_of(gt);
  B200_REQUIRE(pred.data && gt.data && counts, E_INVALID, "overlap_counts: null pointer");
  B200_REQUIRE(pf >= 0, E_UNSUPPORTED, "overlap_counts: prediction kind %d with dtype %d is not supported", pred.kind, pred.dtype);
  B200_REQUIRE(gf >= 0 && (gt.kind == OV_KIND_ONEHOT || gt.kind == OV_KIND_LABEL), E_UNSUPPORTED,
               "overlap_counts: target kind %d with dtype %d is not supported (one-hot uint8 / fp32 or label map uint8 / int64)",
               gt.kind, gt.dtype);
  B200_REQUIRE(C >= 1 && C <= B200_OVERLAP_MAX_CLASSES, E_UNSUPPORTED, "overlap_counts: %d classes; 1..%d are supported", C,
               B200_OVERLAP_MAX_CLASSES);
  B200_REQUIRE(B >= 1 && B <= B200_OVERLAP_MAX_ITEMS, E_UNSUPPORTED, "overlap_counts: %d items; 1..%d per call (one grid row each)",
               B, B200_OVERLAP_MAX_ITEMS);
  B200_REQUIRE(D >= 1 && H >= 1 && W >= 1, E_INVALID, "overlap_counts: d, h, w must be >= 1 (got %d, %d, %d)", D, H, W);
  const long long S = (long long)D * H * W;
  B200_REQUIRE(S < (1LL << 31), E_UNSUPPORTED, "overlap_counts: d*h*w = %lld voxels per item; at most 2^31 - 1", S);
  auto* out = reinterpret_cast<unsigned long long*>(counts);
  B200_CHECK_CUDA(cudaMemsetAsync(out, 0, sizeof(int64_t) * 3 * (size_t)B * C, st));
  switch (pf) {
    case OV_ONEHOT_U8: launch_gt<OV_ONEHOT_U8>(gf, pred, gt, B, C, S, out, st); break;
    case OV_ONEHOT_F32: launch_gt<OV_ONEHOT_F32>(gf, pred, gt, B, C, S, out, st); break;
    case OV_LABEL_U8: launch_gt<OV_LABEL_U8>(gf, pred, gt, B, C, S, out, st); break;
    case OV_LABEL_I64: launch_gt<OV_LABEL_I64>(gf, pred, gt, B, C, S, out, st); break;
    case OV_THRESH_F32: launch_gt<OV_THRESH_F32>(gf, pred, gt, B, C, S, out, st); break;
    default: launch_gt<OV_ARGMAX_F32>(gf, pred, gt, B, C, S, out, st); break;
  }
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

}  // namespace b200
