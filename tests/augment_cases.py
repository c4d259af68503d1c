"""Launch geometry of the training-side input kernels (csrc/augment.cu: k_aug_resample, k_aug_stats, k_aug_apply; csrc/
foreground.cu: the radix select k_fg_hist / k_fg_scan, k_fg_box, k_fg_compose), the regimes the training configurations put them
in, and the GPU cases.

Regime keys:
  - ("resample", source, CM, blocks, last block, padding)
      source: "batch" (launch_augment_resample: the batch on the output grid) or "samples" (launch_augment_resample_samples:
        per-sample pointers and extents, augment.cu:61-64);
      CM: the channel template, 4 for C <= 4 else 16 (augment.cu:209-213);
      blocks: "capped" when ceil(S / 2048) > 1024, so each block walks more than 2048 voxels (aug_blocks, :24-27, :52);
      last block: "partial" when the last block's range is shorter than the others (:52-54), else "whole";
      padding: "border" or "zeros" (:202, :208).
  - ("stats", chain): k_aug_stats over nb partials per (n, c); "several" when nb > 256, so a thread adds several partials
      before the tree (:139-141), else "one".
  - ("intensity", path, grid): k_aug_apply; path "vec4" (S % 4 == 0 and a 16-byte aligned image, :246), "scalar" (S % 4 != 0)
      or "unaligned" (S % 4 == 0, image not 16-byte aligned); grid "capped" when the chunks per plane exceed 132 * 8 / (N C)
      rounded up (:241-244), else "uncapped".
  - ("fg-hist", blocks, idle) and ("fg-box", blocks, samples, idle): the grids of launch_foreground_box's blocks(rows)
      (foreground.cu:269-273), rows = N C planes for k_fg_hist and N samples for k_fg_box; blocks "uncapped", "capped" (the
      cap binds and is above 1) or "one-per-row" (the cap is 1 block per plane or sample); idle "idle" when some sample's range
      split leaves blocks past its end (v0 >= S: the early return at :64, :191), else "busy"; samples "one" or "several".
  - ("select", pass): the radix-select pass at which the keys of the two ranks numpy interpolates between first differ
      (then k_fg_hist keeps two histograms in the later passes, :68-71, :91-92), or "none" when the keys are equal.

The functions below restate the launch code; tests/test_augment_cases_host.py reads the launch constants from the sources,
derives the keys of the configurations in config_sections() and requires a case for every one; tests/test_gpu_augment_kernels.py
runs the cases against fp64 and numpy.  Line numbers refer to 3dunetcnn_b200/csrc/augment.cu for the aug_* rules and to
3dunetcnn_b200/csrc/foreground.cu for the fg_* rules.
"""
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np

# launch constants, read back from the sources by the host test: (file, name) -> value
AUG_THREADS = 256            # kAugThreads (augment.cu:19)
AUG_MAX_BLOCKS = 1024        # kAugMaxBlocks (:20)
AUG_VOXELS_PER_BLOCK = 2048  # kAugVoxelsPerBlock (:21)
AUG_INTENSITY_CAP = 132 * 8  # blocks of k_aug_apply over all planes (:242)
AUG_MAX_CHANNELS = 16        # B200_AUG_MAX_CHANNELS (kernels.h)
FG_THREADS = 256             # kFgThreads (foreground.cu:17)
FG_BINS = 2048               # kFgBins (:18)
FG_UNROLL = 4                # kFgUnroll (:19)
FG_TARGET_BLOCKS = 132 * 8   # kFgTargetBlocks (:20)
SOURCE_CONSTANTS = {
    ("augment.cu", "kAugThreads"): AUG_THREADS, ("augment.cu", "kAugMaxBlocks"): AUG_MAX_BLOCKS,
    ("augment.cu", "kAugVoxelsPerBlock"): AUG_VOXELS_PER_BLOCK, ("foreground.cu", "kFgThreads"): FG_THREADS,
    ("foreground.cu", "kFgBins"): FG_BINS, ("foreground.cu", "kFgUnroll"): FG_UNROLL,
    ("foreground.cu", "kFgTargetBlocks"): FG_TARGET_BLOCKS,
}
U32 = 2.0 ** -24             # fp32 unit roundoff
U64 = 2.0 ** -53             # fp64 unit roundoff


def cdiv(a, b):
    return -(-a // b)


def vol(dims):
    return int(dims[0]) * int(dims[1]) * int(dims[2])


# ------------------------------------------------------------------------------------------------------------ augment.cu
def aug_blocks(S):
    """blocks per sample of k_aug_resample = partial slots per (n, c) (aug_blocks, :24-27)"""
    return min(max(cdiv(S, AUG_VOXELS_PER_BLOCK), 1), AUG_MAX_BLOCKS)


def aug_block_ranges(S):
    """[v0, v1) of each block of one sample: per = ceil(S / gridDim.x) (:51-54); a block past the end gets an empty range"""
    nb = aug_blocks(S)
    per = cdiv(S, nb)
    return [(b * per, min(b * per + per, S)) for b in range(nb)]


def aug_cm(C):
    """the channel template of k_aug_resample (:209-213)"""
    return 4 if C <= 4 else AUG_MAX_CHANNELS


def resample_geometry(S):
    nb = aug_blocks(S)
    per = cdiv(S, nb)
    return dict(nb=nb, per=per, capped=cdiv(S, AUG_VOXELS_PER_BLOCK) > AUG_MAX_BLOCKS, partial=S - (nb - 1) * per < per,
                # longest fp64 addition chain of a partial: per / 256 strided adds, 5 butterfly levels, 8 warp sums (:78-127)
                block_chain=cdiv(per, AUG_THREADS) + 5 + AUG_THREADS // 32,
                # of a statistic over the partials: nb / 256 strided adds, then a tree of log2(256) = 8 levels (:139-150)
                stats_chain=cdiv(nb, AUG_THREADS) + 8)


def resample_key(source, C, out_dims, padding):
    g = resample_geometry(vol(out_dims))
    return ("resample", source, aug_cm(C), "capped" if g["capped"] else "uncapped", "partial" if g["partial"] else "whole", padding)


def stats_key(S):
    return ("stats", "several" if aug_blocks(S) > AUG_THREADS else "one")


def intensity_launch(N, C, S, offset_bytes=0):
    """k_aug_apply's grid and path (launch_augment_intensity, :241-247); offset_bytes: the image's address modulo 16"""
    raw = cdiv(cdiv(S, 4), AUG_THREADS * 4)
    cap = cdiv(AUG_INTENSITY_CAP, N * C)
    chunks = max(min(raw, cap), 1)
    path = "scalar" if S % 4 else ("vec4" if offset_bytes % 16 == 0 else "unaligned")
    return dict(chunks=chunks, capped=raw > cap, path=path)


def intensity_key(N, C, S, offset_bytes=0):
    g = intensity_launch(N, C, S, offset_bytes)
    return ("intensity", g["path"], "capped" if g["capped"] else "uncapped")


# ---------------------------------------------------------------------------------------------------------- foreground.cu
def fg_blocks(max_spatial, rows):
    """blocks(rows) of launch_foreground_box (:269-273): (grid x, regime)"""
    b = cdiv(max_spatial, FG_THREADS * FG_UNROLL * 8)
    cap = cdiv(FG_TARGET_BLOCKS, rows)
    grid = max(min(b, cap), 1)
    return grid, ("one-per-row" if cap == 1 and b > 1 else "capped" if b > cap else "uncapped")


def fg_idle(sizes, grid):
    """some sample leaves blocks with nothing to do: per = ceil(S / grid) and a block starts at or past S (:61-64, :188-191)"""
    return any((grid - 1) * cdiv(s, grid) >= s for s in sizes)


def hist_key(sizes, C):
    grid, regime = fg_blocks(max(sizes), len(sizes) * C)
    return ("fg-hist", regime, "idle" if fg_idle(sizes, grid) else "busy")


def box_key(sizes):
    grid, regime = fg_blocks(max(sizes), len(sizes))
    return ("fg-box", regime, "one" if len(sizes) == 1 else "several", "idle" if fg_idle(sizes, grid) else "busy")


FG_SHIFT = (21, 10, 0)       # digit of pass 0, 1, 2: key bits 31..21, 20..10, 9..0 (fg_shift, :23)
FG_BITS = (11, 11, 10)       # (fg_bits, :24)


def fg_mask(p):
    """key bits fixed before pass p (:68)"""
    return 0 if p == 0 else ~((1 << (FG_SHIFT[p] + FG_BITS[p])) - 1) & 0xFFFFFFFF


def fg_key(x):
    """fp32 -> uint32 in float order, -0 as +0 (fg_key, :45-49)"""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).copy()
    u[u == 0x80000000] = 0
    neg = (u & 0x80000000) != 0
    return np.where(neg, ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def fg_value(k):
    k = np.asarray(k, dtype=np.uint32)
    return np.where((k & 0x80000000) != 0, k ^ np.uint32(0x80000000), ~k).astype(np.uint32).view(np.float32)


def divergence_pass(k_lo, k_hi):
    """the first pass whose digit differs between the two keys, or "none" """
    for p in range(3):
        d = (1 << FG_BITS[p]) - 1
        if (int(k_lo) >> FG_SHIFT[p]) & d != (int(k_hi) >> FG_SHIFT[p]) & d:
            return p
    return "none"


def percentile_index(size, q):
    """np.percentile(x, q * 100)'s ranks and fp32 weight for fp32 data of ``size`` elements (numpy's _quantile "linear",
    restated from augment.percentile_index): (lower rank, upper rank, weight)"""
    qf = np.true_divide(q * 100, np.float32(100))                  # a Python float over fp32: fp32
    vi = (size - 1) * qf
    if vi >= size - 1:
        return size - 1, size - 1, np.float32(vi - np.float32(-1))
    if vi < 0:
        return 0, 0, np.float32(vi)
    prev = int(np.floor(vi))
    return prev, prev + 1, np.float32(vi - np.float32(prev))


def lerp32(a, b, g):
    """k_fg_scan's interpolation (:165-168) = numpy's _lerp in fp32"""
    a, b, g = np.float32(a), np.float32(b), np.float32(g)
    with np.errstate(invalid="ignore", over="ignore"):
        diff = np.float32(b - a)
        return np.float32(b - diff * np.float32(np.float32(1) - g)) if g >= np.float32(0.5) else np.float32(a + diff * g)


def radix_select(x, lo, hi, gamma):
    """numpy restatement of the three passes of k_fg_hist / k_fg_scan (:55-172) on one plane: per pass the histogram of the
    digit of the keys carrying each rank's prefix (one histogram while the prefixes agree), then the bin holding each rank.
    Returns (thr, the passes that kept two histograms)."""
    x = np.asarray(x, dtype=np.float32).reshape(-1)
    nan = bool(np.isnan(x).any())
    k = fg_key(x[~np.isnan(x)]).astype(np.int64)
    pre, rk, two_at = [0, 0], [lo, hi], []
    for p in range(3):
        mask, d = fg_mask(p), (1 << FG_BITS[p]) - 1
        two = pre[0] != pre[1]
        if two:
            two_at.append(p)
        hists = [np.bincount((k[(k & mask) == pre[t]] >> FG_SHIFT[p]) & d, minlength=FG_BINS) for t in range(2 if two else 1)]
        for t in range(2):
            cum = np.cumsum(hists[t if two else 0])
            b = int(np.searchsorted(cum, rk[t], side="right"))
            if b < FG_BINS:                                   # else: the rank is not in the plane (all NaN); kept as it is
                rk[t] -= int(cum[b - 1]) if b else 0
                pre[t] |= b << FG_SHIFT[p]
    v = lerp32(fg_value(np.uint32(pre[0])), fg_value(np.uint32(pre[1])), gamma)
    return (np.float32(np.nan) if nan else v), two_at


def select_pass(x, q):
    """the ("select", pass) regime of one plane at percentile q: where the two ranks' keys diverge"""
    x = np.asarray(x, dtype=np.float32).reshape(-1)
    x = x[~np.isnan(x)]
    if x.size == 0:
        return "none"
    lo, hi, _ = percentile_index(x.size, q)
    s = np.sort(fg_key(x))
    return divergence_pass(s[lo], s[hi])


# ------------------------------------------------------------------------------------------------------------ configurations
# the "dataset" sections of the reference's examples/brats2020/brats2020_config.json and examples/sppin/sppin_config.json with
# their models' in_channels, labels channels after one-hot / hierarchy, batch size and file extents (BraTS 240 x 240 x 155;
# SPPIN 256 x 256 x 160 stored (h, w, d), reoriented to 160 x 256 x 256, sizes differing per item), and the 2 x 4 x 128^3 batch
# that bench.py and the device-transform tests augment without the geometry stage (SPPIN's augmentation lists on a 128^3 batch)
_SPPIN_TRAINING = {
    "spatial_augmentations": [{"name": "RandFlipD", "spatial_axis": 0, "prob": 0.5},
                              {"name": "RandFlipD", "spatial_axis": 1, "prob": 0.5},
                              {"name": "RandRotateD", "prob": 0.5, "range_x": 0.2, "range_y": 0.2, "range_z": 0.2}],
    "intensity_augmentations": [{"name": "RandScaleIntensityD", "factors": 0.1, "prob": 1.0},
                                {"name": "RandShiftIntensityD", "offsets": 0.1, "prob": 1.0}],
}


def config_sections():
    """(name, dataset section, geometry, batch, image channels, label channels, per-sample extents)"""
    brats = {"name": "SegmentationDataset", "desired_shape": [128, 128, 128], "labels": [2, 1, 4], "setup_label_hierarchy": True,
             "normalization": "NormalizeIntensityD", "normalization_kwargs": {"channel_wise": True, "nonzero": False},
             "resample": True, "crop_foreground": True}
    sppin = {"name": "SegmentationDatasetPersistent", "desired_shape": [192, 192, 192], "labels": [1], "orientation": "RAS",
             "normalization": "NormalizeIntensityD", "normalization_kwargs": {"channel_wise": True, "nonzero": False},
             "resample": True, "crop_foreground": True, "foreground_percentile": 0.9, "training": _SPPIN_TRAINING}
    batch = {"normalization_kwargs": {"channel_wise": True}, "training": _SPPIN_TRAINING}
    return [("brats", brats, True, 1, 4, 3, [(240, 240, 155)]),
            ("sppin", sppin, True, 2, 4, 1, [(160, 256, 256), (152, 240, 248)]),
            ("batch-2x4x128", batch, False, 2, 4, 3, [(128, 128, 128)] * 2)]


def config_keys(aug):
    """{key: (config, ...)} of every launch build_device_transform's Compose makes for each configuration (aug: the package's
    augment module).  A percentile threshold whose two ranks differ can diverge at any pass, so it needs every select regime."""
    keys = {}
    for name, section, geometry, n, c, nl, sizes in config_sections():
        comp, _ = aug.build_device_transform(section, geometry=geometry)
        out = comp.resize.spatial_size if comp.resize is not None else sizes[0]
        S = vol(out)
        ks = [resample_key("samples" if geometry else "batch", c, out, comp.padding_mode), intensity_key(n, c, S)]
        if comp.normalize is not None:
            ks.append(stats_key(S))
        if comp.crop is not None:
            ks += [hist_key([vol(s) for s in sizes], c), box_key([vol(s) for s in sizes])]
            if comp.crop.percentile is not None:
                lo, hi, _ = percentile_index(min(vol(s) for s in sizes), comp.crop.percentile)
                ks += [("select", p) for p in ((0, 1, 2, "none") if lo != hi else ("none",))]
        for k in ks:
            keys.setdefault(k, []).append(name)
    return keys


# ------------------------------------------------------------------------------------------------------------ cases
@dataclass(frozen=True)
class ResampleCase:
    """k_aug_resample through b200unet_augment_resample (source "batch") or _resample_samples ("samples"), then the z-score
    and intensity pass over its output.  angles / flips: the rotation and flips drawn on the output grid; samples: the
    per-sample source extents (the map then crops and resizes each one onto ``out``)."""
    id: str
    source: str
    n: int
    c: int
    l: int
    out: Tuple[int, int, int]
    padding: str
    angles: Tuple[float, float, float] = (0.0, 0.0, 0.0)
    flips: Tuple[int, ...] = ()
    samples: Tuple[Tuple[int, int, int], ...] = ()
    nonzero: bool = False
    channel_wise: bool = True
    tagged: Tuple = ()

    @property
    def key(self):
        return resample_key(self.source, self.c, self.out, self.padding)


R = ResampleCase
RESAMPLE_CASES = [
    # 5 channels: the 16-channel template; 25 x 41 x 31 = 31775 -> 16 blocks of 1986, the last one 1985 long
    R("c5-partial-zeros", "batch", 2, 5, 2, (25, 41, 31), "zeros", angles=(0.15, -0.1, 0.2), flips=(1,), nonzero=True,
      tagged=("resample", "batch", 16, "uncapped", "partial", "zeros")),
    # 8 channels, 21 x 23 x 17 = 8211 -> 5 blocks of 1643, the last one 1639 long
    R("c8-partial-border", "batch", 1, 8, 1, (21, 23, 17), "border", angles=(-0.2, 0.05, 0.1), flips=(0, 2),
      channel_wise=False, tagged=("resample", "batch", 16, "uncapped", "partial", "border")),
    # 16 channels, 16 x 16 x 24 = 6144 = 3 x 2048: whole blocks
    R("c16-whole-border", "batch", 2, 16, 0, (16, 16, 24), "border", angles=(0.1, 0.2, -0.15),
      tagged=("resample", "batch", 16, "uncapped", "whole", "border")),
    # above the block cap: 144 x 128 x 128 = 2359296 = 1152 x 2048 -> 1024 blocks of 2304 voxels, none partial
    R("capped-2x2x144x128x128", "batch", 2, 2, 1, (144, 128, 128), "border", angles=(0.12, -0.08, 0.18), flips=(0,),
      tagged=("resample", "batch", 4, "capped", "whole", "border")),
    # 130 x 128 x 129 = 2146560: 1049 blocks of 2048 capped to 1024 of 2097, the last one 1329 long
    R("capped-partial-zeros", "batch", 1, 3, 1, (130, 128, 129), "zeros", angles=(-0.15, 0.1, 0.05), nonzero=True,
      tagged=("resample", "batch", 4, "capped", "partial", "zeros")),
    # the 2 x 4 x 128^3 batch: exactly 1024 blocks of 2048
    R("batch-2x4x128", "batch", 2, 4, 3, (128, 128, 128), "border", angles=(0.2, -0.2, 0.1), flips=(1,),
      tagged=("resample", "batch", 4, "uncapped", "whole", "border")),
    # per-sample sources of different extents: BraTS-like crop + resize onto 64^3 (= 128 x 2048), 4 channels
    R("samples-brats-like", "samples", 1, 4, 3, (64, 64, 64), "border", samples=((75, 70, 50),),
      tagged=("resample", "samples", 4, "uncapped", "whole", "border")),
    # SPPIN-like: two sizes resized onto 144 x 128 x 128, above the cap, with the rotation
    R("samples-capped", "samples", 2, 1, 1, (144, 128, 128), "border", angles=(0.1, 0.15, -0.2), flips=(0,),
      samples=((100, 90, 80), (150, 140, 120)), tagged=("resample", "samples", 4, "capped", "whole", "border")),
    # 6 channels per sample, zeros padding, 19 x 23 x 29 = 12673 -> 7 blocks of 1811, the last one 1807 long
    R("samples-c6-zeros", "samples", 3, 6, 2, (19, 23, 29), "zeros", angles=(0.2, 0.0, 0.1),
      samples=((30, 20, 25), (12, 40, 33), (7, 9, 11)), tagged=("resample", "samples", 16, "uncapped", "partial", "zeros")),
]


@dataclass(frozen=True)
class IntensityCase:
    """k_aug_stats + k_aug_apply through b200unet_augment_intensity on an image written directly (partials filled from it):
    offset = floats between a 16-byte boundary and the image"""
    id: str
    n: int
    c: int
    dims: Tuple[int, int, int]
    offset: int = 0
    normalize: bool = True
    nonzero: bool = False
    channel_wise: bool = True
    tagged: Tuple = ()

    @property
    def key(self):
        return intensity_key(self.n, self.c, vol(self.dims), 4 * self.offset)


I = IntensityCase
INTENSITY_CASES = [
    # S = 7 x 9 x 11 = 693, S % 4 = 1: the scalar path, aligned and one float past a boundary
    I("scalar-aligned", 2, 3, (7, 9, 11), tagged=("intensity", "scalar", "uncapped")),
    I("scalar-offset", 2, 3, (7, 9, 11), offset=1, nonzero=True, tagged=("intensity", "scalar", "uncapped")),
    # S % 4 = 2 and several chunks per plane: 50 x 41 x 31 = 63550, 16 chunks
    I("scalar-chunks", 1, 2, (50, 41, 31), normalize=False, tagged=("intensity", "scalar", "uncapped")),
    # S % 4 == 0, one float off: the scalar loop on a multiple of 4
    I("unaligned-offset", 2, 2, (16, 20, 24), offset=1, channel_wise=False, tagged=("intensity", "unaligned", "uncapped")),
    I("vec4-uncapped", 2, 2, (16, 20, 24), tagged=("intensity", "vec4", "uncapped")),
    # N C = 1100 > 1056 planes: the cap is one block per plane; S = 4 x 32 x 33 = 4224, S % 4 == 0, 2 chunks wanted
    I("vec4-capped-one-block", 100, 11, (4, 32, 33), tagged=("intensity", "vec4", "capped")),
    # the same cap on the scalar path: 5 x 27 x 31 = 4185, S % 4 = 1
    I("scalar-capped-one-block", 100, 11, (5, 27, 31), nonzero=True, tagged=("intensity", "scalar", "capped")),
    # 300 x 64 x 64 = 1228800 = 600 x 2048: 600 partials per (n, c), three per k_aug_stats thread before the tree
    I("stats-several", 1, 2, (300, 64, 64), tagged=("intensity", "vec4", "uncapped")),
]


@dataclass(frozen=True)
class ForegroundCase:
    """launch_foreground_box through b200unet_foreground_box on MRI-like samples (zero background, a core, integer ties)"""
    id: str
    c: int
    sizes: Tuple[Tuple[int, int, int], ...]
    percentile: Optional[float]
    out: Tuple[int, int, int] = (16, 16, 16)
    margin: int = 1
    allow_smaller: bool = True
    tagged: Tuple = ()

    @property
    def keys(self):
        S = [vol(s) for s in self.sizes]
        return (hist_key(S, self.c) if self.percentile is not None else None, box_key(S))


F = ForegroundCase
FOREGROUND_CASES = [
    # BraTS: 1 x 4 x 240 x 240 x 155 at the 10th percentile: 1090 blocks wanted, 264 per plane (hist), 1056 (box)
    F("brats", 4, ((240, 240, 155),), 0.1, out=(128, 128, 128),
      tagged=(("fg-hist", "capped", "busy"), ("fg-box", "capped", "one", "busy"))),
    # SPPIN-like: two sizes at the 90th percentile; the larger wants 565 blocks, 132 per plane, 528 per sample
    F("sppin-like", 4, ((120, 200, 190), (118, 196, 200)), 0.9, out=(32, 32, 32),
      tagged=(("fg-hist", "capped", "busy"), ("fg-box", "capped", "several", "busy"))),
    # 67 x 16 = 1072 planes: one block per plane for the histograms though 9240 voxels want 2; the box grid is 16 blocks
    F("planes-1072", 16, ((20, 21, 22),) * 67, 0.5, out=(8, 8, 8), allow_smaller=False,
      tagged=(("fg-hist", "one-per-row", "busy"), ("fg-box", "uncapped", "several", "busy"))),
    # 1100 samples of one channel: one block per sample for the boxes too
    F("samples-1100", 1, ((9, 30, 31),) * 1100, None, out=(4, 4, 4),
      tagged=(None, ("fg-box", "one-per-row", "several", "busy"))),
    # a mixed-size list: 6.4M voxels want 782 blocks (capped to 132 per plane, 264 per sample); the small ones leave most idle
    F("mixed-sizes", 2, ((200, 200, 160), (3, 4, 5), (1, 1, 1), (17, 1, 29)), 0.25, out=(12, 12, 12),
      tagged=(("fg-hist", "capped", "idle"), ("fg-box", "capped", "several", "idle"))),
    # small volumes, grid 1: the x > 0 mask (no percentile) and boxes past the volume
    F("small-x-gt-0", 3, ((9, 12, 7), (5, 13, 11)), None, margin=2, allow_smaller=False,
      tagged=(None, ("fg-box", "uncapped", "several", "busy"))),
]


@dataclass(frozen=True)
class SelectCase:
    """one plane whose two ranks at ``percentile`` hold chosen values: build() returns fp32 [n]"""
    id: str
    n: int
    percentile: float
    lo_val: float
    hi_val: float
    fill: str = "spread"      # "spread": other values spread around; "zeros": mostly exact zeros; "signed-zeros"; "nan"
    tagged: object = None

    def build(self):
        return select_data(self)


def select_data(case):
    """values below lo_val before the lower rank, at least hi_val after the upper one, shuffled with a fixed seed"""
    g = np.random.default_rng([case.n] + [ord(ch) for ch in case.id])
    n, (lo, hi, _) = case.n, percentile_index(case.n, case.percentile)
    lo_v, hi_v = np.float32(case.lo_val), np.float32(case.hi_val)
    below = lo
    above = n - hi - 1
    if case.fill == "zeros":                                  # heavy ties at the ranks themselves
        x = np.zeros(n, dtype=np.float32)
        x[:below // 2] = -np.abs(g.standard_normal(below // 2)).astype(np.float32) - 1
        x[n - above // 3:] = np.abs(g.standard_normal(above // 3)).astype(np.float32) + 1
    else:
        lo_f = np.float32(-1e30) if np.isinf(lo_v) else lo_v
        hi_f = np.float32(1e30) if np.isinf(hi_v) else hi_v
        span = np.float32(max(1.0, abs(float(lo_f)), abs(float(hi_f))))
        small = (lo_f - span * np.abs(g.random(below)).astype(np.float32) - np.float32(1e-3) * span).astype(np.float32)
        large = (hi_f + span * g.random(above).astype(np.float32)).astype(np.float32)
        if case.fill == "signed-zeros":                       # lo_val = -0 and hi_val = +0 among a run of both
            small[-min(below, 500):] = np.where(g.random(min(below, 500)) < 0.5, -0.0, 0.0)
            large[:min(above, 500)] = np.where(g.random(min(above, 500)) < 0.5, -0.0, 0.0)
        if np.isinf(lo_v):
            small[:] = lo_v
        if np.isinf(hi_v):
            large[:] = hi_v
        x = np.concatenate([small, [lo_v] * (hi - lo + 1 if lo == hi else 1), [] if lo == hi else [hi_v], large]).astype(np.float32)
    if case.fill != "zeros":
        assert x.size == n
    x = g.permutation(x)
    if case.fill == "nan":
        x[n // 3] = np.nan
    return x


S_ = SelectCase
ONE = np.float32(1.0)
SELECT_CASES = [
    # the two ranks differ in sign: the prefixes part at pass 0, two histograms in passes 1 and 2
    S_("div-pass0", 50003, 0.371, -0.5, 0.75, tagged=0),
    # 1 and 1 + 2^-12 share key bits 31..21 and differ in 20..10: two histograms in pass 2
    S_("div-pass1", 40000, 0.61, 1.0, 1.0 + 2.0 ** -12, tagged=1),
    # 1 and the next float: the same prefix until the last digit; negative: the float below -1 and -1 (keys 0x407ffffe, 0x407fffff)
    S_("div-pass2", 33333, 0.2, 1.0, float(np.nextafter(ONE, np.float32(2))), tagged=2),
    S_("div-pass2-negative", 65536, 0.83, float(np.nextafter(-ONE, np.float32(-2))), -1.0, tagged=2),
    # the two ranks on one value
    S_("no-divergence", 30001, 0.45, 2.5, 2.5, tagged="none"),
    # -0 and +0 at the two ranks take one key
    S_("signed-zeros", 20000, 0.5, -0.0, 0.0, fill="signed-zeros", tagged="none"),
    # mostly exact zeros: both ranks inside the run of zeros
    S_("zero-ties", 70000, 0.1, 0.0, 0.0, fill="zeros", tagged="none"),
    # the median of an even count: weight 0.5 exactly, where numpy takes b - (b - a)(1 - t); 0.1 + 0.6 * 0.5 rounds below 0.4
    S_("median-even", 40000, 0.5, 0.1, 0.7, tagged=0),
    # +-inf at the ranks: inf - inf in the interpolation gives NaN, as numpy's
    S_("inf-ranks", 20001, 0.3, float("-inf"), float("inf"), tagged=0),
    S_("inf-upper", 20000, 0.999, 3.0, float("inf"), tagged=0),
    # rank 0 and rank n - 1
    S_("rank-0", 25000, 0.0, -7.25, -7.25, tagged="none"),
    S_("rank-last", 25000, 1.0, 9.5, 9.5, tagged="none"),
    # a NaN anywhere: thr = NaN
    S_("nan", 9000, 0.5, 0.25, 0.5, fill="nan", tagged=0),
]
