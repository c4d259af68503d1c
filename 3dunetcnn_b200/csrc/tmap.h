// Host-side TMA tensor-map construction (cuTensorMapEncodeTiled through cudaGetDriverEntryPoint,
// so the library has no link-time dependency on libcuda).
#pragma once
#include "common.cuh"

namespace b200 {

enum Swz { SWZ_NONE = 0, SWZ_32 = 1, SWZ_64 = 2, SWZ_128 = 3 };

// 5-D map over an NDHWC bf16 view: dims (C, W, H, D, N).  box = (boxC, boxW, boxH, boxD, 1) elements *loaded*;
// estride = traversal stride on the three spatial dims (1, or 2 for the stride-2 convolutions).
// vD/vH/vW (optional): "visible" spatial extents <= D/H/W.  Strides still come from D/H/W, but coordinates at or beyond
// the visible extent read as zero (TMA out-of-bounds fill) - used to mask the padded boundary of a transposed convolution.
int make_act_map(CUtensorMap* out, const bf16* ptr, int N, int D, int H, int W, int C, int ld, int boxC, int boxW,
                 int boxH, int boxD, int estride, Swz swz, int vD = 0, int vH = 0, int vW = 0);

// 5-D map over ONE PARITY CLASS (pd, ph, pw) of an NDHWC view with even extents: logical dims (C, W/2, H/2, D/2, N), element
// (c, w, h, d, n) = tensor[n][2d+pd][2h+ph][2w+pw][c].  Used to TMA-store the output tiles of the stride-2 data gradient
// (one implicit GEMM per output parity class) straight into their interleaved positions.
int make_act_map_class(CUtensorMap* out, const bf16* ptr, int N, int D, int H, int W, int C, int ld, int pd, int ph, int pw,
                       int boxC, int boxW, int boxH, int boxD, Swz swz);

// The two W-parity classes (pd, ph, 0) and (pd, ph, 1) together: logical dims (C, W, H/2, D/2, N) -- W dense, so that a store box
// of 2 * boxW_class voxels per row writes whole 128-byte lines (64-byte pieces of single-class stores land in different lines:
// a profile of the level-0 stride-2 gradient showed one extra DRAM read of the whole output).
int make_act_map_classpair(CUtensorMap* out, const bf16* ptr, int N, int D, int H, int W, int C, int ld, int pd, int ph, int boxC,
                           int boxW, int boxH, int boxD, Swz swz);

// 3-D map over packed weights [T][R][K] bf16 (K contiguous): dims (K, R, T); box (boxK, boxR, 1).
int make_w_map(CUtensorMap* out, const bf16* ptr, int T, int R, int K, int boxK, int boxR, Swz swz, int boxT = 1);

static inline Swz swz_for_bytes(int bytes) { return bytes >= 128 ? SWZ_128 : bytes >= 64 ? SWZ_64 : SWZ_32; }

}  // namespace b200
