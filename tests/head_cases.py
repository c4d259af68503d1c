"""Launch geometry of the tensor-core head for 9..128 outputs (csrc/head.cu: k_head_mma forward, k_head_bwd_mma backward and
the k_sum_slots reduction of csrc/elementwise.cu), the shapes the configurations give it, and the GPU cases.

Regime keys:
  - forward:  ("fwd", NT, tiles per CTA, spread, last tile, samples, epilogue, bias, precision)
  - backward: ("bwd", NT, tiles per CTA, spread, last tile, samples, dlogits path, dbias, precision)
      NT: ceil(n_out / 16), the template instance (head.cu:403-407);
      tiles per CTA: "one" or "several": a CTA walks tiles t, t + grid, ... (head.cu:111, :252), so with several it prefetches
        the next tile into registers (:116, :270-273), reuses sE / sX across tiles (:112) and carries dw / db in registers;
      spread: "even" when the tiles divide evenly over the CTAs, else "uneven" (some CTAs walk one tile more);
      last tile: "partial" when the voxels (N x S) are not a multiple of 128, else "whole";
      samples: "straddle" when a tile holds voxels of two samples (a sample boundary n S is not a multiple of 128), else "within";
      epilogue: "none", "sigmoid" or "softmax" (act_mode 0 / 1 / 2, :158-180);
      dlogits path: "vec" (float4 loads: S % 4 == 0 and a 16-byte aligned dlogits, :209), "scalar" (S % 4 != 0) or "unaligned"
        (S % 4 == 0 but dlogits is not 16-byte aligned, so the scalar loop runs);
      dbias: the fused bias gradient (want_dbias, :339-354, summed by k_sum_slots at elementwise.cu:859-862).

The functions below restate the launch code, so that tests/test_head_cases_host.py derives the keys of the configurations
listed in config_launches() and requires a case for every one of them; tests/test_gpu_head_kernels.py runs the cases against
fp64.  Line numbers refer to 3dunetcnn_b200/csrc/head.cu unless another file is named.
"""
from dataclasses import dataclass
from typing import Optional, Tuple

KTILE = 128                # voxels per tile (head.cu:20)
KMAXC = 64                 # input channels at most, the K padding of the forward (:22)
BWD_SLOTS = 132            # backward CTAs at most = weight-gradient slots (:23)
FWD_CTAS = 2 * 132         # forward CTAs at most (:380)
U = 2.0 ** -24             # fp32 unit roundoff


def cdiv(a, b):
    return -(-a // b)


def vol(dims):
    return dims[0] * dims[1] * dims[2]


def head_geometry(n_out, c, n, dims, aligned=True):
    """the launch of both kernels for x [n][dims][c] and n_out outputs:
      - NT = ceil(n_out / 16) (:403-407), NP = 16 NT padded outputs (:96), NG = NP rounded up to 64 rows of the backward's
        dlogits tile (:195); ksteps = ceil(C / 16) K steps of the forward, zero-padded when C % 16 != 0 (:98);
      - tiles = ceil(N S / 128) (:105, :206); forward grid min(tiles, 264) (launch_fwd_nt, :378-381) and backward slots
        min(tiles, 132) (bwd_grid, :369-372), both at least 1;
      - warpgroup 1 computes dw only when NP > 64 (:287, :328);
      - the dlogits path of load_g (:209, :222-236)."""
    NT = cdiv(n_out, 16)
    NP = 16 * NT
    S = vol(dims)
    total = n * S
    tiles = cdiv(total, KTILE)
    fwd_grid = max(min(tiles, FWD_CTAS), 1)
    slots = max(min(tiles, BWD_SLOTS), 1)
    return dict(NT=NT, NP=NP, NG=cdiv(NP, 64) * 64, S=S, total=total, tiles=tiles, ksteps=cdiv(c, 16), kpad=c % 16 != 0,
                fwd_grid=fwd_grid, fwd_per_cta=cdiv(tiles, fwd_grid), fwd_even=tiles % fwd_grid == 0,
                slots=slots, bwd_per_cta=cdiv(tiles, slots), bwd_even=tiles % slots == 0,
                partial=total % KTILE != 0, straddle=any((k * S) % KTILE for k in range(1, n)), wg1_dw=NP > 64,
                path=("vec" if aligned else "unaligned") if S % 4 == 0 else "scalar")


ACTS = ("none", "sigmoid", "softmax")


def _common(g, per, even):
    return ("one" if per == 1 else "several", "even" if even else "uneven", "partial" if g["partial"] else "whole",
            "straddle" if g["straddle"] else "within")


def fwd_key(n_out, c, n, dims, act, bias, precision):
    g = head_geometry(n_out, c, n, dims)
    return ("fwd", g["NT"]) + _common(g, g["fwd_per_cta"], g["fwd_even"]) + (act, "bias" if bias else "no-bias", precision)


def bwd_key(n_out, c, n, dims, dbias, precision, aligned=True):
    g = head_geometry(n_out, c, n, dims, aligned)
    return ("bwd", g["NT"]) + _common(g, g["bwd_per_cta"], g["bwd_even"]) + (g["path"], "dbias" if dbias else "no-dbias", precision)


# ------------------------------------------------------------------------------------------------------ configurations
C2 = (2, (128, 128, 128))


def config_launches():
    """(config, direction, args) of every head launch with more than 8 outputs in the configurations:
      - README's head table: the C2 size (2 x 128^3) with 32 channels into the head at 16, 32, 64, 104 and 128 outputs, a
        training step in bf16 and in split precision (UNet3D: no bias; DiceLoss takes the logits, so no epilogue);
      - the multi-class fixtures of tests/test_gpu_many_classes.py (1 x 32^3, base width 8): 24 and 104 outputs in training,
        and the 24-output softmax forward in evaluation;
      - the 104-output machinery there: 2 x 32^3 in bf16 and split, 2 x 16^3 in bf16 (the graphed step);
      - its 104-output sliding window: roi 16^3 with sw_batch_size 4 over a 24 x 20 x 28 volume, 8 windows in two batches
        of 4, forward only;
      - DynUNet with 14 outputs and a bias (2 x 32^3, filters[0] = 16);
      - the plan-smooth rows unet_24out_bw16 (UNet3D, 16 channels, 1 x 32^3) and dyn_24out_dx (DynUNet with its bias,
        filters[0] = 16, 1 x 32^3);
      - SegResNet's three_level_24out case of tests/segresnet_cases.py (biased head, init_filters 8, 1 x 24 x 32 x 40), in bf16
        and in split precision.
    args: fwd (n_out, c, n, dims, act, bias, precision); bwd (n_out, c, n, dims, dbias, precision)."""
    out = []

    def train(name, n_out, c, n, dims, bias, precision):
        out.append((name, "fwd", (n_out, c, n, dims, "none", bias, precision)))
        out.append((name, "bwd", (n_out, c, n, dims, bias, precision)))

    for n_out in (16, 32, 64, 104, 128):
        for precision in ("bf16", "split"):
            train("readme-c2-%d-%s" % (n_out, precision), n_out, 32, C2[0], C2[1], False, precision)
    train("mc24", 24, 8, 1, (32, 32, 32), False, "split")
    train("mc104", 104, 8, 1, (32, 32, 32), False, "split")
    out.append(("mc24-softmax-eval", "fwd", (24, 8, 1, (32, 32, 32), "softmax", False, "split")))
    for precision in ("bf16", "split"):
        train("mc104-machinery-32", 104, 8, 2, (32, 32, 32), False, precision)
    train("mc104-machinery-16", 104, 8, 2, (16, 16, 16), False, "bf16")
    out.append(("mc104-sliding-window", "fwd", (104, 8, 4, (16, 16, 16), "none", False, "split")))
    train("dynunet-14-bias", 14, 16, 2, (32, 32, 32), True, "split")
    train("plan-smooth-unet_24out_bw16", 24, 16, 1, (32, 32, 32), False, "split")
    train("plan-smooth-dyn_24out_dx", 24, 16, 1, (32, 32, 32), True, "split")
    for precision in ("bf16", "split"):
        train("segresnet-three_level_24out-%s" % precision, 24, 8, 1, (24, 32, 40), True, precision)
    return out


KEY_OF = {"fwd": fwd_key, "bwd": bwd_key}


def config_keys():
    """{regime key: [(config, args), ...]}"""
    keys = {}
    for name, direction, args in config_launches():
        keys.setdefault(KEY_OF[direction](*args), []).append((name, args))
    return keys


# ------------------------------------------------------------------------------------------------------------ GPU cases
@dataclass(frozen=True)
class Case:
    """one forward and one backward launch on the same x and weights.
      act / bias: the forward's epilogue and bias; the backward computes the fused bias gradient when bias is set;
      ld: x and dx are channel views [c0, c0 + c) of wider NDHWC tensors with ld channels (None: ld = c);
      offset: dlogits is a contiguous view `offset` floats into its storage;
      positive: x and dlogits are positive, so the weight- and bias-gradient sums have no cancellation and a lost tile
        shows above the accumulation bound where a CTA walks few tiles;
      geo: the regime the row is meant to reach, worked out by hand: (tiles per CTA, spread, last tile, samples) of the
        forward, the same of the backward and its dlogits path.  The host test requires the restated launch code to agree."""
    n_out: int
    c: int
    n: int
    dims: Tuple[int, int, int]
    precision: str
    geo: Tuple[Tuple[str, ...], Tuple[str, ...]]
    act: str = "none"
    bias: bool = False
    ld: Optional[int] = None
    offset: int = 0
    positive: bool = False

    @property
    def geometry(self):
        return head_geometry(self.n_out, self.c, self.n, self.dims, self.offset % 4 == 0)

    @property
    def fwd_key(self):
        return fwd_key(self.n_out, self.c, self.n, self.dims, self.act, self.bias, self.precision)

    @property
    def bwd_key(self):
        return bwd_key(self.n_out, self.c, self.n, self.dims, self.bias, self.precision, self.offset % 4 == 0)

    @property
    def tagged_keys(self):
        """(forward key, backward key) from the hand-worked geo"""
        nt = cdiv(self.n_out, 16)
        return (("fwd", nt) + self.geo[0] + (self.act, "bias" if self.bias else "no-bias", self.precision),
                ("bwd", nt) + self.geo[1] + ("dbias" if self.bias else "no-dbias", self.precision))

    @property
    def id(self):
        s = "o%d-c%d-n%d-%s-%s-%s" % (self.n_out, self.c, self.n, "x".join(map(str, self.dims)), self.precision, self.act)
        if self.bias:
            s += "-bias"
        if self.ld is not None:
            s += "-ld%d" % self.ld
        if self.offset:
            s += "-off%d" % self.offset
        if self.positive:
            s += "-pos"
        return s


def _c(n_out, c, n, dims, precision, geo, **kw):
    return Case(n_out, c, n, tuple(dims), precision, geo, **kw)


def _geo(fwd, bwd, path):
    return tuple(fwd.split()), tuple(bwd.split()) + (path,)


# hand-worked regimes of the shapes below (tiles = ceil(N S / 128); 264 forward CTAs, 132 backward slots at most)
GEO_C2 = _geo("several uneven whole within", "several uneven whole within", "vec")       # 32768 tiles: 124.1 / 248.2
GEO_32_1 = _geo("one even whole within", "several uneven whole within", "vec")             # 1 x 32^3: 256 tiles
GEO_32_2 = _geo("several uneven whole within", "several uneven whole within", "vec")       # 2 x 32^3: 512 tiles
GEO_16 = _geo("one even whole within", "one even whole within", "vec")                     # 2 or 4 x 16^3: 64 or 128 tiles
GEO_A = _geo("several uneven partial straddle", "several uneven partial straddle", "scalar")
GEO_B = _geo("several even whole within", "several even whole within", "vec")
GEO_D = _geo("several uneven partial straddle", "several uneven partial straddle", "vec")
GEO_8910 = _geo("one even partial straddle", "one even partial straddle", "vec")          # 1440 voxels: 12 tiles
GEO_573 = _geo("one even partial straddle", "one even partial straddle", "scalar")        # 210 voxels: 2 tiles


def _unaligned(geo):
    return geo[0], geo[1][:4] + ("unaligned",)


# the configurations' shapes, as config_launches() lists them
CONFIG_CASES = (
    # README's head table at the C2 size: 32768 tiles, 124 or 125 per forward CTA and 248 or 249 per backward slot
    [_c(n_out, 32, C2[0], C2[1], precision, GEO_C2, positive=True)
     for n_out in (16, 32, 64, 104, 128) for precision in ("bf16", "split")]
    + [
        _c(24, 8, 1, (32, 32, 32), "split", GEO_32_1),                                # mc24
        _c(104, 8, 1, (32, 32, 32), "split", GEO_32_1),                               # mc104
        _c(24, 8, 1, (32, 32, 32), "split", GEO_32_1, act="softmax"),                 # mc24 softmax evaluation
        _c(104, 8, 2, (32, 32, 32), "bf16", GEO_32_2, positive=True),                 # 104-output machinery
        _c(104, 8, 2, (32, 32, 32), "split", GEO_32_2),
        _c(104, 8, 2, (16, 16, 16), "bf16", GEO_16),                                  # graphed step
        _c(104, 8, 4, (16, 16, 16), "split", GEO_16),                                 # sliding window, one batch of 4 windows
        _c(14, 16, 2, (32, 32, 32), "split", GEO_32_2, bias=True, positive=True),     # DynUNet with a bias
        _c(24, 16, 1, (32, 32, 32), "split", GEO_32_1),                               # plan-smooth unet_24out_bw16
        _c(24, 16, 1, (32, 32, 32), "split", GEO_32_1, bias=True),                    # plan-smooth dyn_24out_dx
        # SegResNet three_level_24out: 1 x 24 x 32 x 40, 240 tiles (one per forward CTA; 1 or 2 per backward slot)
        _c(24, 8, 1, (24, 32, 40), "bf16", GEO_32_1, bias=True),
        _c(24, 8, 1, (24, 32, 40), "split", GEO_32_1, bias=True),
    ])

# Beyond the configurations, per NT 1..8: n_out at both ends of its 16-block (16k + 1, 16k + 16; 9 for NT 1), both
# precisions, several tiles per CTA in both directions, every C from 8 to 64, every epilogue x bias combination.
#   A = 2 x 37 x 41 x 29: S = 43993 (odd, so the scalar dlogits path), 688 tiles with a partial last one, tiles straddle
#       the samples; 3 tiles on some forward CTAs (688 = 2 x 264 + 160) and 5 or 6 per backward slot;
#   B = 2 x 32 x 33 x 32: S = 33792 = 264 x 128, 528 tiles: exactly 2 per forward CTA and 4 per backward slot; positive data;
#   D = 3 x 23 x 24 x 25: S = 13800 (S % 4 == 0, not a multiple of 128), 324 tiles: straddles on the vector path.
SHAPE_A = (2, (37, 41, 29))
SHAPE_B = (2, (32, 33, 32))
SHAPE_D = (3, (23, 24, 25))
_COMBOS = [(a, b) for a in ("none", "sigmoid", "softmax") for b in (False, True)]


def _sweep():
    out = []
    i = 0
    for k in range(8):
        lo, hi = (9 if k == 0 else 16 * k + 1), 16 * k + 16
        for j, (n_out, precision) in enumerate(((lo, "bf16"), (hi, "split"), (lo, "split"), (hi, "bf16"))):
            act, bias = _COMBOS[i % len(_COMBOS)]
            c = 8 * (1 + i % 8)
            ld = c + 16 if i % 5 == 2 else None
            if j < 2:
                out.append(_c(n_out, c, SHAPE_A[0], SHAPE_A[1], precision, GEO_A, act=act, bias=bias, ld=ld))
            else:
                out.append(_c(n_out, c, SHAPE_B[0], SHAPE_B[1], precision, GEO_B, act=act, bias=bias, ld=ld, positive=True))
            i += 1
    return out


SWEEP_CASES = _sweep()

EDGE_CASES = [
    # dlogits one float into its storage with S % 4 == 0: the scalar loop must give the aligned run's bits
    _c(104, 32, SHAPE_B[0], SHAPE_B[1], "split", _unaligned(GEO_B), bias=True, offset=1),
    _c(24, 8, 1, (32, 32, 32), "bf16", _unaligned(GEO_32_1), offset=1),
    _c(128, 64, SHAPE_D[0], SHAPE_D[1], "split", _unaligned(GEO_D), bias=True, offset=1, ld=72),
    # S % 4 == 0 with tiles straddling the samples, on the vector path
    _c(40, 24, SHAPE_D[0], SHAPE_D[1], "bf16", GEO_D, act="softmax", bias=True),
    _c(72, 40, SHAPE_D[0], SHAPE_D[1], "split", GEO_D, act="sigmoid", positive=True),
]


def _small():
    """fewer tiles than CTAs, a partial last tile and samples meeting inside a tile: 2 x 8 x 9 x 10 (12 tiles) at every
    (n_out, C) of 9, 16, 24, 104, 128 x 8, 32, 48, 64 in both precisions, and 2 x 5 x 7 x 3 (2 tiles, S % 4 != 0) with
    each epilogue"""
    out = []
    i = 0
    for n_out in (9, 16, 24, 104, 128):
        for c in (8, 32, 48, 64):
            for precision in ("bf16", "split"):
                act, bias = _COMBOS[i % len(_COMBOS)]
                out.append(_c(n_out, c, 2, (8, 9, 10), precision, GEO_8910, act=act, bias=bias, ld=c + 16 if i % 7 == 3 else None))
                i += 1
    for n_out in (9, 104):
        for precision in ("bf16", "split"):
            out.append(_c(n_out, 32, 2, (5, 7, 3), precision, GEO_573))
    for n_out in (9, 24, 128):
        for act in ("sigmoid", "softmax"):
            out.append(_c(n_out, 32, 2, (5, 7, 3), "split", GEO_573, act=act, bias=n_out == 24))
    return out


SMALL_CASES = _small()

CASES = CONFIG_CASES + SWEEP_CASES + EDGE_CASES + SMALL_CASES
