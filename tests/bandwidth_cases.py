"""Launch geometry of the bandwidth-bound kernels of csrc/elementwise.cu, the shapes the plans give them, and one GPU case per
regime.

A regime key is (kernel, c8n class, capped, tail, precision, view):
  - c8n class: the channel count in 8-channel chunks, "pow2" (a power of two up to 32: lanes that share a chunk are a shuffle
    pattern), "npow2" (any other count up to 32) or "wide" (more than 32 chunks);
  - capped: the grid is clamped, so a thread runs more than one sweep of its grid-stride loop;
  - tail: the last sweep is partial (the `if (s < S)` / `s < total` exits run in some threads and not in others);
  - precision: "bf16" (hi) or "split" (hi + lo);
  - view: the operand the plan hands over is a channel slice of a wider buffer.
The functions below restate the launch code, so that a host test (tests/test_bandwidth_cases_host.py) derives the keys of the
C2, C3 and C5 benchmark plans, the BraTS DynUNet plan and the golden configurations, and requires a case for every one of them;
tests/test_gpu_bandwidth_kernels.py runs the cases against fp64.  Line numbers refer to 3dunetcnn_b200/csrc/elementwise.cu.
"""
from dataclasses import dataclass, field
from typing import Tuple

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
    """k_upsample2x_fwd (launch_upsample2x_fwd, :564-572): one thread per 2 x 2 x 2 output block, (D+1)(H+1)(W+1) blocks"""
    c8n = c // 8
    threads = ew_threads_for(c8n)
    vper = threads // c8n
    nblk = (xdims[0] + 1) * (xdims[1] + 1) * (xdims[2] + 1)
    blocks, capped = _clamp((nblk + vper - 1) // vper, (SMS * 8 + n - 1) // n)
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


def regime_key(kernel, n, c, dims, split, view):
    """dims: the extents the kernel's loop runs over (upsampling: of its low-resolution side)"""
    prec = "split" if split else "bf16"
    if kernel == "gn":
        g = gn_geometry(n, c, dims)
    elif kernel == "act_bwd":
        g = act_bwd_geometry(n, c, dims)
    elif kernel == "up_fwd":
        g = upsample_fwd_geometry(n, c, dims)
    elif kernel == "up_bwd":
        g = upsample_bwd_geometry(n, c, dims, split)
        kernel = "up_bwd_" + upsample_bwd_kernel(split, dims)
    elif kernel == "bias_grad":
        g = bias_grad_geometry(n, c, dims)
    elif kernel == "head_bwd":
        g = head_bwd_geometry(n, c, dims)
    else:
        raise ValueError(kernel)
    return (kernel, c8n_class(c), "capped" if g[2] else "uncapped", "tail" if g[3] else "full-sweeps", prec,
            "view" if view else "full")


# ------------------------------------------------------------------------------------------------------ plan shapes
def _half(dims, k):
    return tuple(d >> k for d in dims)


def unet3d_launches(n, n_features, base_width, dims, encoder_blocks=(1, 2, 2, 4), decoder_blocks=None, convT=False, train=True):
    """(kernel, n, c, dims, view) of every launch of the bandwidth kernels in a UNet3D plan (plan.cu: build_unet3d_plan).  The
    widths double per level; each residual block normalises its input and its first convolution's output; a decoder stage runs
    its blocks at the width it receives, then a 1x1x1 convolution to the next width and the x2 up-sampling into the low half of
    the concat buffer (or, with transposed convolutions, the zero insertion whose backward runs bias_grad on that half)."""
    L = len(encoder_blocks)
    decoder_blocks = list(decoder_blocks) if decoder_blocks is not None else list(encoder_blocks)
    widths = [base_width * 2 ** k for k in range(L)]
    ext = [_half(dims, k) for k in range(L)]
    out = []

    def block(cin, c, k):
        out.append(("gn", n, cin, ext[k], False))
        out.append(("gn", n, c, ext[k], False))
    cin = 8 if n_features <= 8 else 16
    for k in range(L):
        for _ in range(encoder_blocks[k]):
            block(cin, widths[k], k)
            cin = widths[k]
    for i in range(L - 1):
        depth = L - 1 - i
        for _ in range(decoder_blocks[i]):
            block(cin, cin, depth)
        out_w = widths[depth - 1]
        if convT:
            if train:
                out.append(("bias_grad", n, out_w, ext[depth - 1], True))
        else:
            out.append(("up_fwd", n, out_w, ext[depth], True))
            if train:
                out.append(("up_bwd", n, out_w, ext[depth], True))
        cin = 2 * out_w
    for _ in range(decoder_blocks[L - 1]):
        block(cin, base_width, 0)
        cin = base_width
    if train:
        out.append(("head_bwd", n, base_width, dims, False))
    return out


def dynunet_launches(n, filters, dims, train=True):
    """DynUNet with post-activation blocks (conv -> InstanceNorm -> LeakyReLU, twice per block) and strides 1, 2, 2, ...: every norm
    at level k has filters[k] channels; the backward runs act_bwd on each (plan.cu: build_dyn_block_bwd)"""
    out = []
    L = len(filters)
    for k in range(L):
        per_level = 4 if k < L - 1 else 2     # encoder and decoder block, two norms each; the bottleneck has one block
        for _ in range(per_level):
            out.append(("gn", n, filters[k], _half(dims, k), False))
            if train:
                out.append(("act_bwd", n, filters[k], _half(dims, k), False))
    out.append(("head_bwd", n, filters[0], dims, False))
    return out


# The configurations whose shapes the GPU cases must cover: the benchmark's C2 (4 channels, 128^3, width 32, batch 2; also with
# transposed convolutions), C3 (160 x 192 x 128), C5 (1 channel, 5 levels [1, 2, 2, 4, 4], width 48, forward of 3 tiles of 128^3),
# the BraTS DynUNet (examples/brats2020/brats2020_config.json: filters 64 .. 384, six levels; a 128^3 patch, batch 2) and the
# golden configurations of tests/golden/recipe.py.  Training plans run in both precisions.
def plan_launches():
    tr = [
        ("C2", unet3d_launches(2, 4, 32, (128, 128, 128))),
        ("C2-convT", unet3d_launches(2, 4, 32, (128, 128, 128), convT=True)),
        ("C3", unet3d_launches(2, 4, 32, (160, 192, 128))),
        ("brats-dynunet", dynunet_launches(2, [64, 96, 128, 192, 256, 384], (128, 128, 128))),
        ("golden-c1-32", unet3d_launches(1, 4, 8, (32, 32, 32))),
        ("golden-c1-64", unet3d_launches(1, 4, 8, (64, 64, 64))),
        ("golden-bw16", unet3d_launches(2, 4, 16, (32, 32, 32))),
        ("golden-convT", unet3d_launches(1, 4, 8, (32, 32, 32), convT=True)),
        ("golden-c5like", unet3d_launches(1, 1, 8, (32, 32, 32), encoder_blocks=(1, 2, 2, 4, 4), decoder_blocks=(1, 1, 1, 1, 1))),
        ("golden-nonpow2", unet3d_launches(1, 4, 8, (24, 32, 40))),
    ]
    infer = [("C5", unet3d_launches(3, 1, 48, (128, 128, 128), encoder_blocks=(1, 2, 2, 4, 4), decoder_blocks=(1, 1, 1, 1, 1),
                                    train=False))]
    for name, launches in tr:
        for split in (False, True):
            for kernel, n, c, dims, view in launches:
                yield name, (kernel, n, c, dims, split, view)
    for name, launches in infer:
        for kernel, n, c, dims, view in launches:
            yield name, (kernel, n, c, dims, False, view)


def plan_keys():
    """{regime key: [(config, launch), ...]} over every plan above"""
    keys = {}
    for name, (kernel, n, c, dims, split, view) in plan_launches():
        keys.setdefault(regime_key(kernel, n, c, dims, split, view), []).append((name, (n, c, dims)))
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
    key = (kernel if kernel != "up_bwd" else "up_bwd_" + upsample_bwd_kernel(split, dims), cls,
           "capped" if capped else "uncapped", "tail" if tail else "full-sweeps", "split" if split else "bf16", "view" if view else "full")
    return BwCase(kernel, n, c, dims, split, view, key, tuple(sorted(opts.items())))


_ = _case
T, F = True, False
# gn: opts g (groups; 0 = C), real (real channels, default c), slope, bwd ("add1", "add2", "scale", "nogamma")
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
]
CASES = GN_CASES + ACT_CASES + UP_FWD_CASES + UP_BWD_CASES + BIAS_CASES + HEAD_BWD_CASES
