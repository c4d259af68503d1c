"""Launch geometry of the kernels just outside the network -- the sigmoid Dice criterion (csrc/dice.cu), the fused Dice +
cross-entropy criterion (csrc/dice_ce.cu), the sliding-window tiling and z-score kernels (csrc/prepost.cu) -- the shapes the
configurations give them, and one GPU case per regime.

Regime keys:
  - dice:    ("dice", channel class, capped, sweeps, path, target)
      capped: chunks = ceil(S / 1024) is clamped to ceil(1056 / (N*C)) (launch_dice_fwd);
      sweeps: "one-sweep" or "multi-sweep" of a thread's grid-stride loop in k_dice_sums;
      path:   "vec" (float4 / uchar4: uint8 target, S % 4 == 0, aligned pointers), "scalar", or "unaligned" (the vector
              conditions on S and the target type hold but a pointer is not aligned, so the scalar loop runs).
  - dice_ce: ("dice_ce", channel class, target kind, activation, ce, tiles per block, last tile, idle threads)
      target kind and activation as check_shape leaves them (one channel: a uint8 label map is the target itself and softmax
      is ignored); ce: the CE term is evaluated (lambda_ce != 0); tiles per block: ceil(tiles / grid_x) is 1 or more, so the
      aI / aP / aT / ace accumulators carry across a block's tiles or not; last tile: S % 128 != 0; idle: 128 % C != 0, so
      phase B leaves 128 - C * (128 / C) threads idle.
  - tiles:   ("tiles", capped, spans, last batch, roi) for one SlidingWindowInferer call
      capped: grid_for clamps the grid of a gather, scatter, count or normalise launch to 2112 blocks; spans: a tile batch
      holds tiles of two samples (k_tiles_scatter's s[0] == n test and a box over several samples); last batch: the job count
      is not a multiple of sw_batch; roi: "clamped" when a volume extent is smaller than the roi.
  - zscore:  ("zscore", capped, nonzero, grouping)
      capped: the chunks per group are ceil(1056 / groups), not ceil(S / 1024) (launch_zscore).
Channel class: "c1", "few" (2..16) or "many" (17..128).

The functions below restate the launch code, so that tests/test_loss_prepost_cases_host.py derives the keys of the
configurations listed in config_launches() and requires a case for every one of them; tests/test_gpu_loss_prepost_kernels.py runs
the cases against fp64.  Line numbers refer to 3dunetcnn_b200/csrc/dice.cu, dice_ce.cu and prepost.cu.
"""
import math
from dataclasses import dataclass, field
from typing import Tuple

import plan_launches as PL

SMS = 132
U = 2.0 ** -24             # fp32 unit roundoff


def cdiv(a, b):
    return -(-a // b)


def vol(dims):
    return dims[0] * dims[1] * dims[2]


def c_class(c):
    return "c1" if c == 1 else "few" if c <= 16 else "many"


# ------------------------------------------------------------------------------------------------------------ dice.cu
def dice_geometry(n, c, S, target, aligned=True):
    """launch_dice_fwd (dice.cu:171-190) and k_dice_sums (:34-67): chunks per (n, c), whether the cap binds, the path, the
    sweeps of a thread's grid-stride loop and the fp32 chain: the terms a thread adds into aI / aP / aT before the fp64 block
    sum (4 per vector iteration)"""
    chunks = max(cdiv(S, 1024), 1)
    cap = cdiv(SMS * 8, n * c)
    capped = chunks > cap
    if capped:
        chunks = max(cap, 1)
    vec_shape = target == "u8" and S % 4 == 0
    path = ("vec" if aligned else "unaligned") if vec_shape else "scalar"
    items = S // 4 if path == "vec" else S
    sweeps = cdiv(items, chunks * 256)
    return dict(chunks=chunks, capped=capped, path=path, sweeps=sweeps, chain=sweeps * (4 if path == "vec" else 1))


def dice_key(n, c, S, target, aligned=True):
    g = dice_geometry(n, c, S, target, aligned)
    return ("dice", c_class(c), "capped" if g["capped"] else "uncapped", "one-sweep" if g["sweeps"] == 1 else "multi-sweep",
            g["path"], target)


# ---------------------------------------------------------------------------------------------------------- dice_ce.cu
KV = 128                   # voxels per tile (dice_ce.cu:29)
KTHREADS = 128
KP = KV + 1
SMEM_PER_SM = 228 * 1024
SMEM_RESERVED = 1024
TARGET_KINDS = {"label_u8": 0, "label_i64": 1, "onehot_u8": 2, "soft_f32": 3}


def dice_ce_effective(c, kind, act):
    """check_shape (dice_ce.cu:362-367): with one channel a uint8 label map is the one-hot target and softmax is ignored"""
    if c == 1:
        if kind == "label_u8":
            kind = "onehot_u8"
        if act == "softmax":
            act = None
    return kind, act


def tile_smem(c, kind):
    """tile_smem (:52-56)"""
    b = 8 * KTHREADS * 3 + 4 * c * KP
    if TARGET_KINDS[kind] >= TARGET_KINDS["onehot_u8"]:
        b += 4 * c * KP
    return b + 4 * KV + 4 * KV


def grid_x(n, c, S, kind):
    """grid_x (:59-67): blocks per sample"""
    tiles = cdiv(S, KV)
    per_sm = max(min(SMEM_PER_SM // (tile_smem(c, kind) + SMEM_RESERVED), 2048 // KTHREADS), 1)
    return max(min(cdiv(SMS * per_sm, n), tiles), 1)


def dice_ce_geometry(n, c, S, kind, act):
    kind, act = dice_ce_effective(c, kind, act)
    gx = grid_x(n, c, S, kind)
    K = KTHREADS // c
    # phase B (:168-182): thread (c, slice) adds voxels slice, slice + K, ... of a tile in two interleaved fp32 chains, then
    # adds them into its fp64 accumulators
    chain = cdiv(cdiv(KV, K), 2) + 1
    return dict(kind=kind, act=act, smem=tile_smem(c, kind), grid_x=gx, tiles=cdiv(S, KV), tiles_per_block=cdiv(cdiv(S, KV), gx),
                K=K, idle=KTHREADS - K * c, chain=chain)


def dice_ce_key(n, c, S, kind, act, with_ce):
    g = dice_ce_geometry(n, c, S, kind, act)
    return ("dice_ce", c_class(c), g["kind"], g["act"] or "none", "ce" if with_ce else "no-ce",
            "multi-tile" if g["tiles_per_block"] > 1 else "one-tile", "partial-tile" if S % KV else "whole-tiles",
            "idle" if g["idle"] else "no-idle")


# ---------------------------------------------------------------------------------------------------------- prepost.cu
def grid_for(total, block=256):
    """grid_for (prepost.cu:103-107): (blocks, capped)"""
    g = cdiv(total, block)
    cap = SMS * 16
    return (max(g, 1) if g <= cap else cap), g > cap


def scan_starts(size, roi, overlap):
    """predict.py: _scan_starts"""
    interval = max(int(roi * (1 - overlap)), 1)
    if size <= roi:
        return [0]
    k = int(math.ceil(float(size - roi) / interval)) + 1
    return [min(i * interval, size - roi) for i in range(k)]


def tiling_plan(shape, roi, overlap, sw_batch):
    """SlidingWindowInferer.__call__: the roi clamped to the volume, the jobs (sample, d0, h0, w0) in order and the batches"""
    n, _, D, H, W = shape
    r = tuple(min(a, b) for a, b in zip(roi, (D, H, W)))
    axes = [scan_starts(s, q, overlap) for s, q in zip((D, H, W), r)]
    jobs = [(b, d, h, w) for b in range(n) for d in axes[0] for h in axes[1] for w in axes[2]]
    return r, axes, jobs, [jobs[j:j + sw_batch] for j in range(0, len(jobs), sw_batch)]


def scatter_box(batch, r):
    """launch_tiles_scatter (:135-141): the box over the batch's tiles, over all samples"""
    lo = [min(j[k + 1] for j in batch) for k in range(3)]
    hi = [max(j[k + 1] + r[k] for j in batch) for k in range(3)]
    return tuple(h - l for l, h in zip(lo, hi))


def tiling_geometry(shape, roi, overlap, sw_batch, c_out):
    n, c, D, H, W = shape
    r, axes, jobs, batches = tiling_plan(shape, roi, overlap, sw_batch)
    capped = {
        "gather": grid_for(sw_batch * c * vol(r))[1],
        "scatter": any(grid_for(n * c_out * vol(scatter_box(b, r)))[1] for b in batches),
        "count": grid_for(D * H * W)[1],
        "normalize": grid_for(n * c_out * D * H * W)[1],
    }
    spans = any(len({j[0] for j in b}) > 1 for b in batches)
    return dict(roi=r, axes=axes, jobs=len(jobs), batches=len(batches), capped=capped, spans=spans,
                partial=len(jobs) % sw_batch != 0, clamped=any(a < b for a, b in zip((D, H, W), roi)),
                max_cover=math.prod(max(sum(1 for s in a if s <= v < s + q) for v in range(e)) for a, q, e in zip(axes, r, (D, H, W))))


def tiling_key(shape, roi, overlap, sw_batch, c_out):
    g = tiling_geometry(shape, roi, overlap, sw_batch, c_out)
    return ("tiles", "capped" if any(g["capped"].values()) else "uncapped", "spans" if g["spans"] else "within",
            "partial-last" if g["partial"] else "full-last", "clamped" if g["clamped"] else "roi")


def zscore_geometry(groups, S):
    """launch_zscore (:254-256)"""
    chunks = cdiv(SMS * 8, groups)
    per = cdiv(S, 1024)
    capped = chunks <= per
    if chunks > per:
        chunks = max(per, 1)
    return dict(chunks=chunks, capped=capped, sweeps=cdiv(S, chunks * 256))


def zscore_key(c, dims, nonzero, channel_wise):
    groups = c if channel_wise else 1
    g = zscore_geometry(groups, c * vol(dims) // groups)
    return ("zscore", "capped" if g["capped"] else "uncapped", "nonzero" if nonzero else "all",
            "channel-wise" if channel_wise else "whole")


# ------------------------------------------------------------------------------------------------------ configurations
def config_launches():
    """(config, kernel, args) of every criterion / pre- / post-processing launch of the configurations:
      - bench.py C2 (batch 2, 3 outputs, 128^3) and C3 (160 x 192 x 128), the BraTS config (3 sigmoid outputs, batch 2 of
        128^3 patches) and the BraTS SegResNet recipe (3 sigmoid outputs, 1 x 224 x 224 x 144): DiceLoss(sigmoid=True) on uint8
        one-hot targets;
      - the golden recipes (tests/plan_launches.py), and the many-class setups of tests/test_gpu_many_classes.py: the 24- and
        104-output fixtures (1 x 32^3), the 104-output machinery (2 x 32^3 and 2 x 16^3) and the 128-output head shape
        (2 x 5 x 7 x 3);
      - README's head table at the C2 size with 104 and 128 outputs: DiceLoss(sigmoid=True) on uint8 one-hot targets;
      - a DiceCELoss(softmax=True, to_onehot_y=True) step on a label map at 128^3, batch 2, 3 and 16 classes, uint8 and int64;
      - bench.py C5's tiled inference: one 256^3 volume, roi 128^3, overlap 0.25, sw_batch 3, one output channel;
      - the BraTS z-score: NormalizeIntensity(nonzero=True, channel_wise=True) on 4 channels at 128^3 and 240 x 240 x 155."""
    out = []
    for name, (n, c, dims) in [("C2", (2, 3, (128, 128, 128))), ("C3", (2, 3, (160, 192, 128))), ("brats", (2, 3, (128, 128, 128))),
                               ("brats-segresnet", (1, 3, (224, 224, 144)))]:
        out.append((name, "dice", (n, c, vol(dims), "u8")))
    for c in PL.CONFIGS:
        if c.name.startswith("golden-"):          # every one trains on DiceLoss(sigmoid=True), uint8 one-hot
            out.append((c.name, "dice", (c.n, c.kw["n_outputs"], vol(c.dims), "u8")))
    for name, (n, c, dims) in [("mc24", (1, 24, (32, 32, 32))), ("mc104", (1, 104, (32, 32, 32))),
                               ("mc104-machinery", (2, 104, (32, 32, 32))), ("mc104-graph", (2, 104, (16, 16, 16))),
                               ("mc128-head", (2, 128, (5, 7, 3)))]:
        out.append((name, "dice", (n, c, vol(dims), "u8")))
    for c in (104, 128):
        out.append(("C2-%d" % c, "dice", (2, c, 128 ** 3, "u8")))
    for c in (3, 16):
        for kind in ("label_u8", "label_i64"):
            out.append(("dicece-label-c%d" % c, "dice_ce", (2, c, 128 ** 3, kind, "softmax", True)))
    out.append(("C5", "tiles", ((1, 1, 256, 256, 256), (128, 128, 128), 0.25, 3, 1)))
    for dims in ((128, 128, 128), (240, 240, 155)):
        out.append(("brats-zscore", "zscore", (4, dims, True, True)))
    return out


KEY_OF = {"dice": dice_key, "dice_ce": dice_ce_key, "tiles": tiling_key, "zscore": zscore_key}


def config_keys():
    """{regime key: [(config, args), ...]}"""
    keys = {}
    for name, kernel, args in config_launches():
        keys.setdefault(KEY_OF[kernel](*args), []).append((name, args))
    return keys


# ------------------------------------------------------------------------------------------------------------ GPU cases
@dataclass(frozen=True)
class Case:
    """one launch; args are those of the kernel's key function, key the regime it must reach (the host test recomputes it).
    opts: options of the GPU test."""
    kernel: str
    args: tuple
    key: Tuple[str, ...]
    opts: Tuple[Tuple[str, object], ...] = field(default=())

    @property
    def opt(self):
        return dict(self.opts)

    @property
    def id(self):
        a = self.args
        if self.kernel == "dice":
            s = "n%d-c%d-s%d-%s" % a[:4] + ("" if len(a) < 5 or a[4] else "-unaligned")
        elif self.kernel == "dice_ce":
            s = "n%d-c%d-s%d-%s-%s-%s" % (a[0], a[1], a[2], a[3], a[4] or "none", "ce" if a[5] else "noce")
        elif self.kernel == "tiles":
            s = "%s-roi%s-ov%g-swb%d-out%d" % ("x".join(map(str, a[0])), "x".join(map(str, a[1])), a[2], a[3], a[4])
        else:
            s = "c%d-%s-%s-%s" % (a[0], "x".join(map(str, a[1])), "nz" if a[2] else "all", "cw" if a[3] else "whole")
        o = "".join("-%s%s" % (k, v) for k, v in self.opts)
        return "%s-%s%s" % (self.kernel, s, o)


def _case(kernel, *args, key, **opts):
    return Case(kernel, tuple(args), tuple(key), tuple(sorted(opts.items())))


T, F = True, False
# dice: args (n, c, S, target[, aligned]); opts: misaligned operand ("target" at storage offset 1, "logits" at one float)
DICE_CASES = [
    _case("dice", 2, 3, 128 ** 3, "u8", key=("dice", "few", "capped", "multi-sweep", "vec", "u8")),                 # C2, BraTS
    _case("dice", 2, 3, 160 * 192 * 128, "u8", key=("dice", "few", "capped", "multi-sweep", "vec", "u8")),          # C3
    _case("dice", 2, 3, 128 ** 3, "f32", key=("dice", "few", "capped", "multi-sweep", "scalar", "f32")),
    _case("dice", 1, 3, 32 ** 3, "u8", key=("dice", "few", "uncapped", "one-sweep", "vec", "u8")),                  # golden
    _case("dice", 1, 3, 24 * 32 * 40, "u8", key=("dice", "few", "uncapped", "one-sweep", "vec", "u8")),
    _case("dice", 2, 3, 32 ** 3, "f32", key=("dice", "few", "uncapped", "multi-sweep", "scalar", "f32")),
    _case("dice", 2, 3, 12 * 10 * 16, "u8", key=("dice", "few", "uncapped", "one-sweep", "vec", "u8")),
    _case("dice", 2, 3, 5 * 7 * 3, "u8", key=("dice", "few", "uncapped", "one-sweep", "scalar", "u8")),
    _case("dice", 2, 3, 9 * 10 * 11, "f32", key=("dice", "few", "uncapped", "multi-sweep", "scalar", "f32")),
    _case("dice", 2, 3, 61 * 50 * 45, "u8", key=("dice", "few", "uncapped", "multi-sweep", "scalar", "u8")),
    _case("dice", 1, 1, 32 ** 3, "u8", key=("dice", "c1", "uncapped", "one-sweep", "vec", "u8")),                   # golden C5-like
    _case("dice", 2, 1, 160 ** 3, "u8", key=("dice", "c1", "capped", "multi-sweep", "vec", "u8")),
    _case("dice", 2, 1, 96 ** 3 + 1, "f32", key=("dice", "c1", "capped", "multi-sweep", "scalar", "f32")),
    _case("dice", 1, 24, 32 ** 3, "u8", key=("dice", "many", "uncapped", "one-sweep", "vec", "u8")),                # mc24
    _case("dice", 1, 104, 32 ** 3, "u8", key=("dice", "many", "capped", "multi-sweep", "vec", "u8")),               # mc104
    _case("dice", 2, 104, 32 ** 3, "u8", key=("dice", "many", "capped", "multi-sweep", "vec", "u8")),
    _case("dice", 2, 104, 64 ** 3, "u8", key=("dice", "many", "capped", "multi-sweep", "vec", "u8")),
    # README's head table at the C2 size: 1368 (104 classes) and 1640 (128) terms in a thread's fp32 chains
    _case("dice", 2, 104, 128 ** 3, "u8", key=("dice", "many", "capped", "multi-sweep", "vec", "u8")),              # C2-104
    _case("dice", 2, 128, 128 ** 3, "u8", key=("dice", "many", "capped", "multi-sweep", "vec", "u8")),              # C2-128
    _case("dice", 2, 104, 16 ** 3, "u8", key=("dice", "many", "uncapped", "one-sweep", "vec", "u8")),
    _case("dice", 2, 128, 105, "u8", key=("dice", "many", "uncapped", "one-sweep", "scalar", "u8")),                # mc128 head
    _case("dice", 2, 128, 32 ** 3, "f32", key=("dice", "many", "capped", "multi-sweep", "scalar", "f32")),
    # a contiguous target (or logits) view at a storage offset: the vector conditions on S hold, the pointer is not aligned
    _case("dice", 2, 3, 32 ** 3, "u8", False, key=("dice", "few", "uncapped", "multi-sweep", "unaligned", "u8"), misaligned="target"),
    _case("dice", 2, 3, 128 ** 3, "u8", False, key=("dice", "few", "capped", "multi-sweep", "unaligned", "u8"), misaligned="target"),
    _case("dice", 2, 3, 12 * 10 * 16, "u8", False, key=("dice", "few", "uncapped", "multi-sweep", "unaligned", "u8"), misaligned="logits"),
]
# dice_ce: args (n, c, S, target kind, act, with_ce)
DICE_CE_CASES = [
    _case("dice_ce", 2, 3, 128 ** 3, "label_u8", "softmax", T,
          key=("dice_ce", "few", "label_u8", "softmax", "ce", "multi-tile", "whole-tiles", "idle")),
    _case("dice_ce", 2, 3, 128 ** 3, "label_i64", "softmax", T,
          key=("dice_ce", "few", "label_i64", "softmax", "ce", "multi-tile", "whole-tiles", "idle")),
    _case("dice_ce", 2, 16, 128 ** 3, "label_u8", "softmax", T,
          key=("dice_ce", "few", "label_u8", "softmax", "ce", "multi-tile", "whole-tiles", "no-idle")),
    _case("dice_ce", 2, 16, 128 ** 3, "label_i64", "softmax", T,
          key=("dice_ce", "few", "label_i64", "softmax", "ce", "multi-tile", "whole-tiles", "no-idle")),
    # several tiles per block and a partial last tile, every target form and activation
    _case("dice_ce", 2, 3, 100 * 90 * 77, "label_u8", "softmax", F,
          key=("dice_ce", "few", "label_u8", "softmax", "no-ce", "multi-tile", "partial-tile", "idle")),
    _case("dice_ce", 2, 5, 100 * 90 * 77, "label_i64", "sigmoid", T,
          key=("dice_ce", "few", "label_i64", "sigmoid", "ce", "multi-tile", "partial-tile", "idle")),
    _case("dice_ce", 2, 4, 100 * 90 * 77, "onehot_u8", None, T,
          key=("dice_ce", "few", "onehot_u8", "none", "ce", "multi-tile", "partial-tile", "no-idle")),
    _case("dice_ce", 1, 3, 100 * 90 * 77, "soft_f32", "softmax", T,
          key=("dice_ce", "few", "soft_f32", "softmax", "ce", "multi-tile", "partial-tile", "idle")),
    _case("dice_ce", 2, 1, 100 * 90 * 77, "label_u8", "sigmoid", T,
          key=("dice_ce", "c1", "onehot_u8", "sigmoid", "ce", "multi-tile", "partial-tile", "no-idle")),
    _case("dice_ce", 1, 1, 100 * 90 * 77, "soft_f32", "softmax", F,
          key=("dice_ce", "c1", "soft_f32", "none", "no-ce", "multi-tile", "partial-tile", "no-idle")),
    _case("dice_ce", 2, 104, 40 * 40 * 41, "label_u8", "softmax", T,
          key=("dice_ce", "many", "label_u8", "softmax", "ce", "multi-tile", "partial-tile", "idle")),
    _case("dice_ce", 1, 128, 31 * 32 * 33, "onehot_u8", "sigmoid", F,
          key=("dice_ce", "many", "onehot_u8", "sigmoid", "no-ce", "multi-tile", "partial-tile", "no-idle")),
    # one tile per block (the shapes of tests/test_gpu_dice_ce.py), whole and partial
    _case("dice_ce", 2, 3, 24 * 32 * 40, "label_u8", "softmax", T,
          key=("dice_ce", "few", "label_u8", "softmax", "ce", "one-tile", "whole-tiles", "idle")),
    _case("dice_ce", 2, 3, 5 * 7 * 3, "label_i64", "softmax", T,
          key=("dice_ce", "few", "label_i64", "softmax", "ce", "one-tile", "partial-tile", "idle")),
    _case("dice_ce", 2, 8, 9 * 10 * 11, "onehot_u8", "softmax", T,
          key=("dice_ce", "few", "onehot_u8", "softmax", "ce", "one-tile", "partial-tile", "no-idle")),
    _case("dice_ce", 2, 3, 9 * 10 * 11, "soft_f32", "sigmoid", F,
          key=("dice_ce", "few", "soft_f32", "sigmoid", "no-ce", "one-tile", "partial-tile", "idle")),
    _case("dice_ce", 2, 24, 12 * 10 * 16, "label_u8", None, T,
          key=("dice_ce", "many", "label_u8", "none", "ce", "one-tile", "whole-tiles", "idle")),
]
# tiles: args (input shape, roi, overlap, sw_batch, output channels)
TILE_CASES = [
    _case("tiles", (1, 1, 256, 256, 256), (128, 128, 128), 0.25, 3, 1, key=("tiles", "capped", "within", "full-last", "roi")),   # C5
    _case("tiles", (1, 2, 256, 256, 256), (128, 128, 128), 0.25, 3, 3, key=("tiles", "capped", "within", "full-last", "roi")),
    _case("tiles", (2, 3, 20, 24, 28), (16, 16, 16), 0.25, 5, 2, key=("tiles", "uncapped", "spans", "partial-last", "roi")),
    _case("tiles", (2, 2, 80, 80, 80), (64, 64, 64), 0.25, 3, 3, key=("tiles", "capped", "spans", "partial-last", "roi")),
    _case("tiles", (3, 1, 40, 12, 30), (16, 16, 16), 0.5, 7, 4, key=("tiles", "uncapped", "spans", "partial-last", "clamped")),
    _case("tiles", (2, 2, 20, 24, 28), (16, 16, 16), 0.25, 4, 3, key=("tiles", "uncapped", "within", "full-last", "roi")),
    _case("tiles", (1, 3, 33, 17, 40), (16, 16, 24), 0.25, 5, 3, key=("tiles", "uncapped", "within", "partial-last", "roi")),
    _case("tiles", (1, 1, 12, 40, 12), (16, 16, 16), 0.25, 1, 3, key=("tiles", "uncapped", "within", "full-last", "clamped")),
]
# zscore: args (channels, dims, nonzero, channel_wise)
ZSCORE_CASES = [
    _case("zscore", 4, (128, 128, 128), T, T, key=("zscore", "capped", "nonzero", "channel-wise")),                 # BraTS
    _case("zscore", 4, (240, 240, 155), T, T, key=("zscore", "capped", "nonzero", "channel-wise")),
    _case("zscore", 4, (128, 128, 128), F, T, key=("zscore", "capped", "all", "channel-wise")),
    _case("zscore", 4, (96, 96, 96), T, F, key=("zscore", "capped", "nonzero", "whole")),
    _case("zscore", 4, (20, 24, 28), T, T, key=("zscore", "uncapped", "nonzero", "channel-wise")),
    _case("zscore", 4, (20, 24, 28), F, F, key=("zscore", "uncapped", "all", "whole")),
    _case("zscore", 5, (7, 9, 11), T, T, key=("zscore", "uncapped", "nonzero", "channel-wise")),
]
CASES = DICE_CASES + DICE_CE_CASES + TILE_CASES + ZSCORE_CASES
