"""Launch geometry of the bandwidth-bound kernels of csrc/elementwise.cu, the shapes the plans give them, and one GPU case per
regime.

A regime key is (kernel, c8n class, capped, tail, precision, view):
  - c8n class: the channel count in 8-channel chunks, "pow2" (a power of two up to 32: lanes that share a chunk are a shuffle
    pattern), "npow2" (any other count up to 32) or "wide" (more than 32 chunks);
  - capped: the grid is clamped, so a thread runs more than one sweep of its grid-stride loop;
  - tail: the last sweep is partial (the `if (s < S)` / `s < total` exits run in some threads and not in others);
  - precision: "bf16" (hi) or "split" (hi + lo);
  - view: the operand the plan hands over is a channel slice of a wider buffer.
The SIMT head's forward keys the class of its input width, and its bias gradient (k_head_dbias, which reads only the fp32
dlogits) keys "one-sample" / "batch" in the class slot and "fp32" as its precision.
The functions below restate the launch code, so that a host test (tests/test_bandwidth_cases_host.py) derives the keys of every
plan configuration of tests/plan_launches.py and requires a case for every one of them; tests/test_gpu_bandwidth_kernels.py runs
the cases against fp64.  Line numbers refer to 3dunetcnn_b200/csrc/elementwise.cu.
"""
from dataclasses import dataclass, field
from typing import Tuple

import plan_launches as PL

SMS = 132


def ew_threads_for(c8n):
    """threads per block of the channel-chunked kernels (ew_threads_for, :164)"""
    for t in range(256, 31, -32):
        if t % c8n == 0:
            return t
    return (256 // c8n) * c8n if c8n <= 256 else c8n


def ew_blocks(total, threads):
    """ew_blocks (:157)"""
    b = (total + threads - 1) // threads
    return max(b, 1) if b < SMS * 16 else SMS * 16


def _clamp(want, cap):
    return (max(want, 1) if want < cap else cap), want > cap


def c8n_class(c):
    c8n = c // 8
    if c8n > 32:
        return "wide"
    return "pow2" if c8n & (c8n - 1) == 0 else "npow2"


def vol(dims):
    return dims[0] * dims[1] * dims[2]


def gn_geometry(n, c, dims):
    """k_gn_apply / k_gn_bwd (gn_launch_dims, :172): (blocks, threads, capped, tail); two voxels per thread per step"""
    c8n = c // 8
    threads = ew_threads_for(c8n)
    vper = threads // c8n
    S = vol(dims)
    blocks, capped = _clamp((S + 2 * vper - 1) // (2 * vper), (SMS * 8 + n - 1) // n)
    return blocks, threads, capped, S % (2 * blocks * vper) != 0


def act_bwd_geometry(n, c, dims):
    """k_act_bwd (launch_act_bwd, :418-425)"""
    c8n = c // 8
    threads = ew_threads_for(c8n)
    vper = threads // c8n
    S = vol(dims)
    blocks, capped = _clamp((S + vper - 1) // vper, (SMS * 4 + n - 1) // n)
    return blocks, threads, capped, S % (blocks * vper) != 0


def upsample_fwd_geometry(n, c, xdims):
    """k_upsample2x_fwd (launch_upsample2x_fwd): one thread per 2 x 2 x 2 output block, (D+1)(H+1)(W+1) blocks, at most 4 blocks
    per SM for each sample whatever the batch"""
    c8n = c // 8
    threads = ew_threads_for(c8n)
    vper = threads // c8n
    nblk = (xdims[0] + 1) * (xdims[1] + 1) * (xdims[2] + 1)
    blocks, capped = _clamp((nblk + vper - 1) // vper, SMS * 4)
    return blocks, threads, capped, nblk % (blocks * vper) != 0


def upsample_bwd_kernel(split, xdims):
    """the kernel launch_upsample2x_bwd picks (:706): the register-blocked form for bf16 with even extents >= 2, else the gather"""
    return "blk" if not split and all(d % 2 == 0 and d >= 2 for d in xdims) else "gather"


def upsample_bwd_geometry(n, c, xdims, split):
    c8n = c // 8
    if upsample_bwd_kernel(split, xdims) == "blk":
        total, threads = n * vol(xdims) // 8 * c8n, 128
    else:
        total, threads = n * vol(xdims) * c8n, 256
    blocks = ew_blocks(total, threads)
    return blocks, threads, (total + threads - 1) // threads > SMS * 16, total % (blocks * threads) != 0


def bias_grad_geometry(n, c, dims):
    """k_bias_grad (launch_bias_grad): at most 592 blocks"""
    c8n = c // 8
    threads = ew_threads_for(c8n)
    vper = threads // c8n
    V = n * vol(dims)
    blocks, capped = _clamp((V + vper - 1) // vper, 592)
    return blocks, threads, capped, V % (blocks * vper) != 0


def head_bwd_threads(c):
    """the SIMT head_bwd block size (launch_head_bwd, :869-870): 256 rounded up to a multiple of c8n in steps of 32"""
    t = 256
    while t % (c // 8):
        t += 32
    return t


def head_bwd_geometry(n, c, dims):
    threads = head_bwd_threads(c)
    total = n * vol(dims) * (c // 8)
    blocks = min(ew_blocks(total, threads), 1184)
    return blocks, threads, (total + threads - 1) // threads > 1184, total % (blocks * threads) != 0


def head_fwd_geometry(n, c, dims):
    """k_head_fwd (launch_head_fwd, :776): one thread per voxel of the batch, 256 threads, ew_blocks"""
    total = n * vol(dims)
    blocks = ew_blocks(total, 256)
    return blocks, 256, (total + 255) // 256 > SMS * 16, total % (blocks * 256) != 0


def head_dbias_geometry(n, dims):
    """k_head_dbias (launch_head_dbias, :465-470): per output min(ceil(S / 256), 128) blocks of 256 threads sweep each sample's S
    voxels, the samples one after another"""
    S = vol(dims)
    blocks, capped = _clamp((S + 255) // 256, 128)
    return blocks, 256, capped, S % (blocks * 256) != 0


def regime_key(kernel, n, c, dims, split, view):
    """dims: the extents the kernel's loop runs over (upsampling: of its low-resolution side)"""
    prec = "split" if split else "bf16"
    cls = c8n_class(c)
    if kernel == "gn":
        g = gn_geometry(n, c, dims)
    elif kernel == "act_bwd":
        g = act_bwd_geometry(n, c, dims)
    elif kernel in ("up_fwd", "up_add"):
        g = upsample_fwd_geometry(n, c, dims)
    elif kernel == "up_bwd":
        g = upsample_bwd_geometry(n, c, dims, split)
        kernel = "up_bwd_" + upsample_bwd_kernel(split, dims)
    elif kernel == "bias_grad":
        g = bias_grad_geometry(n, c, dims)
    elif kernel == "head_bwd":
        g = head_bwd_geometry(n, c, dims)
    elif kernel == "head_fwd":
        g = head_fwd_geometry(n, c, dims)
    elif kernel == "head_dbias":
        g = head_dbias_geometry(n, dims)
        cls, prec = ("one-sample" if n == 1 else "batch"), "fp32"
    else:
        raise ValueError(kernel)
    return (kernel, cls, "capped" if g[2] else "uncapped", "tail" if g[3] else "full-sweeps", prec, "view" if view else "full")


# ------------------------------------------------------------------------------------------------------ plan shapes
KERNELS = ("gn", "act_bwd", "up_fwd", "up_add", "up_bwd", "bias_grad", "head_fwd", "head_bwd", "head_dbias")


def plan_launches_by_config():
    """(training plans, forward-only plans): [(config, [launch of a keyed kernel, ...]), ...] over every configuration of
    tests/plan_launches.py"""
    tr, infer = [], []
    for c in PL.CONFIGS:
        (tr if c.train else infer).append((c.name, [l for l in c.launches() if l.kernel in KERNELS]))
    return tr, infer


def plan_gn_bwd_variants():
    """{k_gn_bwd variant: [config, ...]} over the training plans (the regime key does not carry the variant)"""
    out = {}
    for name, launches in plan_launches_by_config()[0]:
        for l in launches:
            if l.variant is not None and name not in out.setdefault(l.variant, []):
                out[l.variant].append(name)
    return out


def plan_keys():
    """{regime key: [(config, launch), ...]} over every plan; training plans run in both precisions"""
    keys = {}
    tr, infer = plan_launches_by_config()
    for plans, precisions in ((tr, (False, True)), (infer, (False,))):
        for name, launches in plans:
            for split in precisions:
                for l in launches:
                    key = regime_key(l.kernel, l.n, PL.pad8(l.c), l.dims, split, l.view)
                    keys.setdefault(key, []).append((name, (l.n, PL.pad8(l.c), l.dims)))
    return keys


# ------------------------------------------------------------------------------------------------------------ GPU cases
@dataclass(frozen=True)
class BwCase:
    """one launch of a keyed kernel: n, c (channels of the view), dims (the extents regime_key takes), precision, view;
    key = the regime it must reach (the host test recomputes it).  opts: kernel-specific options of the GPU test."""
    kernel: str
    n: int
    c: int
    dims: Tuple[int, int, int]
    split: bool
    view: bool
    key: Tuple[str, ...]
    opts: Tuple[Tuple[str, object], ...] = field(default=())

    @property
    def opt(self):
        return dict(self.opts)

    @property
    def id(self):
        o = "".join("-%s%s" % (k, v) for k, v in self.opts)
        return "%s-n%d-c%d-%s-%s%s%s" % (self.kernel, self.n, self.c, "x".join(map(str, self.dims)), "split" if self.split else "bf16",
                                       "-view" if self.view else "", o)


def _case(kernel, n, c, dims, split, view, cls, capped, tail, **opts):
    prec = "fp32" if kernel == "head_dbias" else "split" if split else "bf16"
    key = (kernel if kernel != "up_bwd" else "up_bwd_" + upsample_bwd_kernel(split, dims), cls,
           "capped" if capped else "uncapped", "tail" if tail else "full-sweeps", prec, "view" if view else "full")
    return BwCase(kernel, n, c, dims, split, view, key, tuple(sorted(opts.items())))


_ = _case
T, F = True, False
# gn: opts g (groups; 0 = C), real (real channels, default c), slope, bwd ("plain", "add1", "add1+add2", "add1+scale", "scale",
# "nogamma"), whole (1: add1 is a whole buffer, as SegResNet's ResBlocks hand it over; else a channel slice)
GN_CASES = [
    _("gn", 2, 8, (4, 4, 4), F, F, "pow2", F, T, g=8, bwd="add1"),
    _("gn", 2, 8, (4, 4, 4), T, F, "pow2", F, T, g=8, bwd="add1"),
    _("gn", 2, 16, (8, 12, 8), F, F, "pow2", F, F, g=8, bwd="add1"),
    _("gn", 2, 16, (8, 12, 8), T, F, "pow2", F, F, g=8, bwd="add1"),
    _("gn", 2, 8, (4, 5, 7), F, F, "pow2", F, T, real=4, g=4, bwd="add1"),
    _("gn", 2, 8, (4, 5, 7), T, F, "pow2", F, T, real=4, g=4, bwd="add1"),
    _("gn", 2, 24, (6, 4, 10), F, F, "npow2", F, T, g=8, slope=0.01, bwd="add1+add2"),
    _("gn", 2, 24, (6, 4, 10), T, F, "npow2", F, T, g=0, bwd="scale"),
    _("gn", 2, 32, (48, 48, 48), F, F, "pow2", T, T, g=8, bwd="add1"),
    _("gn", 2, 32, (48, 48, 48), T, F, "pow2", T, T, g=8, slope=0.01, bwd="scale"),
    _("gn", 5, 32, (16, 32, 64), F, F, "pow2", T, T, g=1, bwd="nogamma"),
    _("gn", 1, 48, (32, 32, 32), F, F, "npow2", F, F, g=8, bwd="add1"),
    _("gn", 2, 48, (32, 32, 32), T, F, "npow2", F, F, g=0, slope=0.01, bwd="add1+add2"),
    _("gn", 2, 48, (40, 40, 40), F, F, "npow2", T, T, g=8, bwd="add1"),
    _("gn", 2, 96, (40, 40, 40), T, F, "npow2", T, T, g=0, slope=0.01, bwd="add1"),
    _("gn", 2, 64, (32, 32, 32), F, F, "pow2", F, F, g=8, bwd="add1"),
    _("gn", 2, 64, (32, 32, 32), T, F, "pow2", F, F, g=8, bwd="scale"),
    _("gn", 2, 96, (16, 16, 16), F, F, "npow2", F, F, g=8, slope=0.01, bwd="add1"),
    _("gn", 2, 96, (16, 16, 16), T, F, "npow2", F, F, g=0, bwd="nogamma"),
    _("gn", 2, 96, (5, 6, 7), F, F, "npow2", F, T, g=96, bwd="add1"),
    _("gn", 2, 128, (8, 8, 8), F, F, "pow2", F, F, g=8, bwd="add1"),
    _("gn", 2, 128, (8, 8, 8), T, F, "pow2", F, F, g=8, bwd="add1"),
    _("gn", 2, 192, (16, 16, 16), F, F, "npow2", F, F, g=8, bwd="add1"),
    _("gn", 2, 192, (16, 16, 16), T, F, "npow2", F, F, g=0, slope=0.01, bwd="add1"),
    _("gn", 2, 256, (16, 16, 16), F, F, "pow2", F, F, g=8, bwd="add1"),
    _("gn", 2, 256, (16, 16, 16), T, F, "pow2", F, F, g=8, bwd="add1"),
    _("gn", 2, 256, (8, 8, 8), F, F, "pow2", F, F, g=8, bwd="add1"),
    _("gn", 2, 320, (5, 6, 7), F, F, "wide", F, T, g=8, bwd="add1"),
    _("gn", 2, 384, (16, 16, 16), F, F, "wide", F, F, g=0, slope=0.01, bwd="add1"),
    _("gn", 2, 384, (16, 16, 16), T, F, "wide", F, F, g=8, bwd="add1"),
    _("gn", 2, 384, (4, 4, 4), F, F, "wide", F, F, g=8, bwd="add1"),
    _("gn", 2, 384, (8, 8, 8), T, F, "wide", F, F, g=8, bwd="add1"),
    _("gn", 3, 384, (8, 8, 8), F, F, "wide", F, F, g=8, bwd="add1"),
    _("gn", 2, 768, (16, 16, 16), F, F, "wide", T, T, g=8, bwd="add1"),
    _("gn", 3, 768, (8, 8, 8), F, F, "wide", F, F, g=8, bwd="add1"),
    _("gn", 2, 1024, (17, 16, 16), F, F, "wide", T, T, g=8, slope=0.01, bwd="add1+add2"),
    # SegResNet: the first ResBlock's residual addend and Dropout3d scale together, the other norms without either
    _("gn", 1, 16, (64, 64, 72), F, F, "pow2", T, T, g=8, bwd="add1+scale", whole=1),
    _("gn", 1, 16, (64, 64, 72), T, F, "pow2", T, T, g=8, bwd="add1+scale", whole=1),
    _("gn", 2, 24, (24, 40, 32), T, F, "npow2", F, F, g=8, bwd="add1+scale", whole=1),
    _("gn", 2, 48, (12, 20, 16), F, F, "npow2", F, F, g=8, bwd="plain"),
    _("gn", 1, 16, (64, 64, 72), T, F, "pow2", T, T, g=8, bwd="plain"),
]
# act_bwd: opts g2 (0/1), slope, ld (bstats pitch beyond C)
ACT_CASES = [
    _("act_bwd", 2, 24, (6, 10, 8), T, F, "npow2", F, T, g2=1, slope=0.01),
    _("act_bwd", 2, 24, (6, 10, 8), F, F, "npow2", F, T, g2=1, slope=0.01),
    _("act_bwd", 2, 24, (6, 10, 8), T, F, "npow2", F, T, g2=0, slope=0.0, ld=8),
    _("act_bwd", 2, 32, (24, 32, 32), F, F, "pow2", T, T, g2=1, slope=0.01),
    _("act_bwd", 2, 64, (64, 64, 64), F, F, "pow2", T, T, g2=1, slope=0.01),
    _("act_bwd", 2, 64, (64, 64, 64), T, F, "pow2", T, T, g2=0, slope=0.01),
    _("act_bwd", 2, 64, (5, 6, 7), F, F, "pow2", F, T, g2=0, slope=0.0, ld=16),
    _("act_bwd", 2, 96, (32, 32, 32), F, F, "npow2", T, T, g2=1, slope=0.01),
    _("act_bwd", 2, 96, (32, 32, 32), T, F, "npow2", T, T, g2=0, slope=0.01),
    _("act_bwd", 2, 128, (16, 16, 16), F, F, "pow2", F, F, g2=1, slope=0.01),
    _("act_bwd", 2, 128, (16, 16, 16), T, F, "pow2", F, F, g2=1, slope=0.01),
    _("act_bwd", 2, 192, (8, 8, 8), F, F, "npow2", F, F, g2=1, slope=0.01),
    _("act_bwd", 2, 192, (8, 8, 8), T, F, "npow2", F, F, g2=0, slope=0.01),
    _("act_bwd", 2, 256, (4, 4, 4), F, F, "pow2", F, F, g2=1, slope=0.01),
    _("act_bwd", 2, 256, (4, 4, 4), T, F, "pow2", F, F, g2=0, slope=0.01),
    _("act_bwd", 2, 384, (4, 4, 4), F, F, "wide", F, F, g2=0, slope=0.01),
    _("act_bwd", 2, 384, (4, 4, 4), T, F, "wide", F, F, g2=1, slope=0.0),
]
# up_fwd: opts ld (stats pitch and concat buffer: c + ld channels, the output at channel 8)
UP_FWD_CASES = [
    _("up_fwd", 2, 16, (4, 6, 8), F, T, "pow2", F, T),
    _("up_fwd", 2, 16, (3, 5, 7), F, T, "pow2", F, T),
    _("up_fwd", 2, 16, (3, 5, 7), T, T, "pow2", F, T),
    _("up_fwd", 2, 16, (1, 2, 4), F, T, "pow2", F, T),
    _("up_fwd", 2, 16, (1, 2, 4), T, T, "pow2", F, T),
    _("up_fwd", 2, 16, (2, 2, 6), F, T, "pow2", F, T),
    _("up_fwd", 2, 16, (2, 2, 6), T, T, "pow2", F, T),
    _("up_fwd", 2, 8, (1, 3, 5), F, T, "pow2", F, T),
    _("up_fwd", 2, 16, (4, 6, 8), T, T, "pow2", F, T),
    _("up_fwd", 2, 16, (64, 64, 64), F, T, "pow2", T, T),
    _("up_fwd", 2, 16, (64, 64, 64), T, T, "pow2", T, T),
    _("up_fwd", 2, 32, (32, 32, 32), F, T, "pow2", T, T),
    _("up_fwd", 2, 32, (32, 32, 32), T, T, "pow2", T, T),
    _("up_fwd", 2, 64, (16, 16, 16), F, T, "pow2", F, T),
    _("up_fwd", 2, 64, (16, 16, 16), T, T, "pow2", F, T),
    _("up_fwd", 2, 128, (8, 8, 8), F, T, "pow2", F, T),
    _("up_fwd", 2, 128, (8, 8, 8), T, T, "pow2", F, T),
    _("up_fwd", 2, 256, (3, 5, 2), F, T, "pow2", F, F),
    _("up_fwd", 2, 256, (3, 5, 2), T, T, "pow2", F, F),
    _("up_fwd", 1, 8, (8, 8, 8), F, T, "pow2", F, T),
    _("up_fwd", 1, 8, (8, 8, 8), T, T, "pow2", F, T),
    _("up_fwd", 2, 24, (3, 1, 5), F, T, "npow2", F, T),
    _("up_fwd", 2, 48, (5, 4, 3), T, T, "npow2", F, T),
    _("up_fwd", 3, 48, (32, 32, 32), F, T, "npow2", T, T),
    _("up_fwd", 3, 96, (16, 16, 16), F, T, "npow2", F, T),
    _("up_fwd", 3, 192, (8, 8, 8), F, T, "npow2", F, T),
    _("up_fwd", 2, 192, (4, 3, 5), T, T, "npow2", F, F),
    _("up_fwd", 3, 384, (4, 4, 4), F, T, "wide", F, T),
    _("up_fwd", 2, 768, (3, 2, 3), F, T, "wide", F, F),
]
# up_add: the fused up-sampling + skip-add into a whole buffer (SegResNet's decoder)
UP_ADD_CASES = [
    _("up_add", 1, 16, (56, 56, 44), F, F, "pow2", T, T),
    _("up_add", 1, 32, (56, 56, 36), T, F, "pow2", T, T),
    _("up_add", 1, 64, (28, 28, 18), F, F, "pow2", F, T),
    _("up_add", 1, 64, (28, 28, 18), T, F, "pow2", F, T),
    _("up_add", 2, 48, (6, 10, 8), F, F, "npow2", F, T),
    _("up_add", 2, 96, (3, 5, 4), T, F, "npow2", F, T),
    _("up_add", 2, 24, (12, 20, 16), T, F, "npow2", F, T),
    _("up_add", 1, 24, (40, 40, 44), T, F, "npow2", T, T),
]
UP_BWD_CASES = [
    _("up_bwd", 2, 16, (3, 5, 7), T, T, "pow2", F, T),
    _("up_bwd", 2, 16, (1, 2, 4), T, T, "pow2", F, T),
    _("up_bwd", 2, 16, (2, 2, 6), T, T, "pow2", F, T),
    _("up_bwd", 2, 16, (4, 6, 8), F, T, "pow2", F, T),
    _("up_bwd", 2, 16, (2, 2, 6), F, T, "pow2", F, T),
    _("up_bwd", 2, 16, (3, 5, 7), F, T, "pow2", F, T),
    _("up_bwd", 2, 16, (1, 2, 4), F, T, "pow2", F, T),
    _("up_bwd", 2, 16, (4, 6, 8), T, T, "pow2", F, F),
    _("up_bwd", 2, 32, (64, 64, 64), F, T, "pow2", F, F),
    _("up_bwd", 2, 32, (64, 64, 64), T, T, "pow2", T, T),
    _("up_bwd", 2, 32, (64, 64, 80), F, T, "pow2", T, T),
    _("up_bwd", 1, 64, (3, 4, 5), T, T, "pow2", F, T),
    _("up_bwd", 2, 64, (32, 32, 32), F, T, "pow2", F, F),
    _("up_bwd", 2, 64, (32, 32, 32), T, T, "pow2", F, F),
    _("up_bwd", 2, 128, (16, 16, 16), F, T, "pow2", F, F),
    _("up_bwd", 2, 128, (16, 16, 16), T, T, "pow2", F, F),
    _("up_bwd", 1, 8, (16, 16, 16), F, T, "pow2", F, F),
    _("up_bwd", 1, 8, (16, 16, 16), T, T, "pow2", F, F),
    _("up_bwd", 1, 16, (8, 8, 8), F, T, "pow2", F, F),
    _("up_bwd", 1, 32, (4, 4, 4), F, T, "pow2", F, T),
    _("up_bwd", 2, 24, (4, 6, 2), F, T, "npow2", F, T),
    _("up_bwd", 2, 48, (3, 1, 5), F, T, "npow2", F, T),
    _("up_bwd", 2, 384, (2, 4, 2), F, T, "wide", F, T),
    # SegResNet: dy is a whole C-channel buffer
    _("up_bwd", 1, 32, (56, 56, 36), F, F, "pow2", F, F),
    _("up_bwd", 1, 64, (28, 28, 18), F, F, "pow2", F, T),
    _("up_bwd", 2, 48, (6, 10, 8), F, F, "npow2", F, T),
    _("up_bwd", 1, 16, (64, 64, 72), T, F, "pow2", T, T),
    _("up_bwd", 1, 64, (28, 28, 18), T, F, "pow2", F, F),
    _("up_bwd", 1, 16, (6, 8, 10), T, F, "pow2", F, T),
    _("up_bwd", 2, 24, (12, 20, 16), T, F, "npow2", F, F),
    _("up_bwd", 2, 96, (3, 5, 4), F, F, "npow2", F, T),
    _("up_bwd", 2, 96, (3, 5, 4), T, F, "npow2", F, T),
]
BIAS_CASES = [
    _("bias_grad", 2, 32, (128, 128, 128), F, T, "pow2", T, T),
    _("bias_grad", 2, 32, (128, 128, 128), T, T, "pow2", T, T),
    _("bias_grad", 2, 64, (32, 32, 32), F, T, "pow2", T, T),
    _("bias_grad", 2, 64, (32, 32, 32), T, T, "pow2", T, T),
    _("bias_grad", 2, 128, (16, 16, 16), F, T, "pow2", F, F),
    _("bias_grad", 2, 128, (16, 16, 16), T, T, "pow2", F, F),
    _("bias_grad", 1, 8, (32, 32, 32), F, T, "pow2", F, F),
    _("bias_grad", 1, 8, (32, 32, 32), T, T, "pow2", F, F),
    _("bias_grad", 1, 16, (16, 16, 16), F, T, "pow2", F, F),
    _("bias_grad", 1, 16, (16, 16, 16), T, T, "pow2", F, F),
    _("bias_grad", 1, 32, (8, 8, 8), F, T, "pow2", F, F),
    _("bias_grad", 1, 32, (8, 8, 8), T, T, "pow2", F, F),
    _("bias_grad", 2, 40, (5, 6, 9), F, T, "npow2", F, T),
    _("bias_grad", 2, 256, (5, 6, 9), T, T, "pow2", F, T),
]
# head_bwd: opts o (outputs)
HEAD_BWD_CASES = [
    _("head_bwd", 2, 32, (6, 6, 10), T, F, "pow2", F, T, o=3),
    _("head_bwd", 2, 32, (128, 128, 128), F, F, "pow2", T, T, o=3),
    _("head_bwd", 2, 32, (128, 128, 128), T, F, "pow2", T, T, o=2),
    _("head_bwd", 2, 64, (128, 128, 128), F, F, "pow2", T, T, o=3),
    _("head_bwd", 2, 64, (128, 128, 128), T, F, "pow2", T, T, o=1),
    _("head_bwd", 1, 8, (32, 32, 32), F, F, "pow2", F, F, o=5),
    _("head_bwd", 1, 8, (32, 32, 32), T, F, "pow2", F, F, o=4),
    _("head_bwd", 1, 8, (64, 64, 64), F, F, "pow2", F, F, o=6),
    _("head_bwd", 1, 8, (64, 64, 64), T, F, "pow2", F, F, o=7),
    _("head_bwd", 2, 16, (32, 32, 32), F, F, "pow2", F, F, o=8),
    _("head_bwd", 2, 16, (32, 32, 32), T, F, "pow2", F, F, o=3),
    _("head_bwd", 2, 48, (5, 6, 7), F, F, "npow2", F, T, o=3),
    _("head_bwd", 2, 24, (6, 6, 10), T, F, "npow2", F, T, o=2),
    _("head_bwd", 2, 32, (6, 6, 10), F, F, "pow2", F, T, o=3),
    _("head_bwd", 2, 8, (6, 6, 10), F, F, "pow2", F, T, o=8),
    _("head_bwd", 2, 24, (24, 40, 32), F, F, "npow2", F, F, o=5),
    _("head_bwd", 2, 24, (24, 40, 32), T, F, "npow2", F, F, o=5),
]
# head_fwd (1..8 outputs): opts o (outputs)
HEAD_FWD_CASES = [
    _("head_fwd", 1, 32, (64, 96, 96), F, F, "pow2", T, T, o=3),
    _("head_fwd", 1, 16, (64, 96, 96), T, F, "pow2", T, T, o=3),
    _("head_fwd", 1, 48, (64, 96, 96), F, F, "npow2", T, T, o=1),
    _("head_fwd", 1, 8, (32, 32, 32), F, F, "pow2", F, F, o=3),
    _("head_fwd", 1, 8, (32, 32, 32), T, F, "pow2", F, F, o=2),
    _("head_fwd", 2, 24, (24, 40, 32), F, F, "npow2", F, F, o=5),
    _("head_fwd", 2, 24, (24, 40, 32), T, F, "npow2", F, F, o=5),
]
# head_dbias: c is not read; opts o (outputs)
HEAD_DBIAS_CASES = [
    _("head_dbias", 1, 16, (224, 224, 144), F, F, "one-sample", T, T, o=3),
    _("head_dbias", 1, 8, (32, 32, 32), F, F, "one-sample", F, F, o=2),
    _("head_dbias", 2, 64, (128, 128, 128), F, F, "batch", T, F, o=3),
    _("head_dbias", 2, 16, (32, 32, 48), F, F, "batch", T, T, o=3),
    _("head_dbias", 2, 24, (24, 40, 32), F, F, "batch", F, F, o=5),
]
CASES = (GN_CASES + ACT_CASES + UP_FWD_CASES + UP_ADD_CASES + UP_BWD_CASES + BIAS_CASES + HEAD_BWD_CASES + HEAD_FWD_CASES
         + HEAD_DBIAS_CASES)
