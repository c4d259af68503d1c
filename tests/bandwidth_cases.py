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
The functions below restate the launch code, so that a host test (tests/test_bandwidth_cases_host.py) derives the keys of the
C2, C3 and C5 benchmark plans, the BraTS DynUNet and SegResNet plans, the SegResNet plan cases and the golden configurations, and
requires a case for every one of them; tests/test_gpu_bandwidth_kernels.py runs the cases against fp64.  Line numbers refer to
3dunetcnn_b200/csrc/elementwise.cu.
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
def _half(dims, k):
    return tuple(d >> k for d in dims)


def unet3d_launches(n, n_features, base_width, dims, encoder_blocks=(1, 2, 2, 4), decoder_blocks=None, convT=False, train=True):
    """(kernel, n, c, dims, view[, GroupNorm backward variant]) of every launch of the bandwidth kernels in a UNet3D plan (plan.cu:
    build_unet3d_plan).  The widths double per level; each residual block normalises its input and its first convolution's output;
    a decoder stage runs its blocks at the width it receives, then a 1x1x1 convolution to the next width and the x2 up-sampling into
    the low half of the concat buffer (or, with transposed convolutions, the zero insertion whose backward runs bias_grad on that
    half).  The head has no bias.  The variant (training plans) is what build_block_bwd hands k_gn_bwd: "plain", "add1" (the
    block's output gradient as the residual addend, when the block keeps its width) or "add1+scale" (and the Dropout3d scale); the
    network's first norm runs no k_gn_bwd (None)."""
    L = len(encoder_blocks)
    decoder_blocks = list(decoder_blocks) if decoder_blocks is not None else list(encoder_blocks)
    widths = [base_width * 2 ** k for k in range(L)]
    ext = [_half(dims, k) for k in range(L)]
    out = []

    def block(cin, c, k, first=False, scale_in=False):
        v1 = None if first else "plain" if cin != c else "add1+scale" if scale_in else "add1"
        out.append(("gn", n, cin, ext[k], False, v1 if train else None))
        out.append(("gn", n, c, ext[k], False, "plain" if train else None))
    cin = 8 if n_features <= 8 else 16
    for k in range(L):
        for b in range(encoder_blocks[k]):
            block(cin, widths[k], k, first=k == 0 and b == 0, scale_in=k == 0 and b == 1)
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
    out.append(("head_fwd", n, base_width, dims, False))
    if train:
        out.append(("head_bwd", n, base_width, dims, False))
    return out


def dynunet_launches(n, filters, dims, train=True):
    """DynUNet with post-activation blocks (conv -> InstanceNorm -> LeakyReLU, twice per block) and strides 1, 2, 2, ...: every norm
    at level k has filters[k] channels; the backward runs act_bwd on each and k_gn_bwd without addend or scale (plan.cu:
    build_dyn_block_bwd).  The head has a bias."""
    out = []
    L = len(filters)
    for k in range(L):
        per_level = 4 if k < L - 1 else 2     # encoder and decoder block, two norms each; the bottleneck has one block
        for _ in range(per_level):
            out.append(("gn", n, filters[k], _half(dims, k), False, "plain" if train else None))
            if train:
                out.append(("act_bwd", n, filters[k], _half(dims, k), False))
    out.append(("head_fwd", n, filters[0], dims, False))
    if train:
        out.append(("head_bwd", n, filters[0], dims, False))
        out.append(("head_dbias", n, filters[0], dims, False))
    return out


def segresnet_launches(n, F, dims, blocks_down=(1, 2, 2, 4), blocks_up=(1, 1, 1), train=True, dropout=True):
    """SegResNet (plan.cu: build_segresnet): level i has F << i channels; every ResBlock normalises its input and its first
    convolution's output, both whole buffers, and in the backward hands its output gradient to the first norm's k_gn_bwd as the
    residual addend (the first encoder block also the Dropout3d scale of convInit's output, when dropout is on).  A decoder stage
    runs the 1x1x1 convolution to C channels at the lower level's extents, then the fused x2 up-sampling + skip-add (up_add, a
    whole C-channel output), its blocks, and in the backward the up-sampling's adjoint from the whole C-channel gradient.  The
    head normalises F channels (act_bwd on it alone) and runs the biased 1x1x1 convolution."""
    L = len(blocks_down)
    ext = [_half(dims, k) for k in range(L)]
    out = []

    def block(c, k, scale_in=False):
        out.append(("gn", n, c, ext[k], False, ("add1+scale" if scale_in else "add1") if train else None))
        out.append(("gn", n, c, ext[k], False, "plain" if train else None))
    for i in range(L):
        for b in range(blocks_down[i]):
            block(F << i, i, scale_in=dropout and i == 0 and b == 0)
    for i in range(L - 1):
        j = L - 2 - i
        out.append(("up_add", n, F << j, ext[j + 1], False))
        for _ in range(blocks_up[i]):
            block(F << j, j)
        if train:
            out.append(("up_bwd", n, F << j, ext[j + 1], False))
    out.append(("gn", n, F, dims, False, "plain" if train else None))
    out.append(("head_fwd", n, F, dims, False))
    if train:
        out.append(("act_bwd", n, F, dims, False))
        out.append(("head_bwd", n, F, dims, False))
        out.append(("head_dbias", n, F, dims, False))
    return out


def _segresnet_case_launches(case):
    """segresnet_launches of a tests/segresnet_cases.py plan case"""
    bd, bu = case.blocks
    return segresnet_launches(case.shape[0], case.kw.get("init_filters", 8), case.shape[2:], bd, bu,
                              dropout=case.dropout or case.kw.get("dropout_prob", 0.0) > 0)


# The configurations whose shapes the GPU cases must cover: the benchmark's C2 (4 channels, 128^3, width 32, batch 2; also with
# transposed convolutions), C3 (160 x 192 x 128), C5 (1 channel, 5 levels [1, 2, 2, 4, 4], width 48, forward of 3 tiles of 128^3),
# the BraTS DynUNet (examples/brats2020/brats2020_config.json: filters 64 .. 384, six levels; a 128^3 patch, batch 2), the BraTS
# SegResNet recipe (init_filters 16, blocks_down [1, 2, 2, 4], blocks_up [1, 1, 1], dropout 0.2: training at 1 x 224 x 224 x 144
# and 2 x 128^3, the two shapes tools/segresnet_bench.py times, and its forward-only plan), the SegResNet plan cases of
# tests/segresnet_cases.py and the golden configurations of tests/golden/recipe.py.  Training plans run in both precisions.
def plan_launches_by_config():
    import segresnet_cases as SC
    brats = dict(blocks_down=(1, 2, 2, 4), blocks_up=(1, 1, 1))
    tr = [
        ("C2", unet3d_launches(2, 4, 32, (128, 128, 128))),
        ("C2-convT", unet3d_launches(2, 4, 32, (128, 128, 128), convT=True)),
        ("C3", unet3d_launches(2, 4, 32, (160, 192, 128))),
        ("brats-dynunet", dynunet_launches(2, [64, 96, 128, 192, 256, 384], (128, 128, 128))),
        ("brats-segresnet", segresnet_launches(1, 16, (224, 224, 144), **brats)),
        ("brats-segresnet-128", segresnet_launches(2, 16, (128, 128, 128), **brats)),
        ("brats-segresnet-infer", segresnet_launches(1, 16, (224, 224, 144), train=False, **brats)),
        ("golden-c1-32", unet3d_launches(1, 4, 8, (32, 32, 32))),
        ("golden-c1-64", unet3d_launches(1, 4, 8, (64, 64, 64))),
        ("golden-bw16", unet3d_launches(2, 4, 16, (32, 32, 32))),
        ("golden-convT", unet3d_launches(1, 4, 8, (32, 32, 32), convT=True)),
        ("golden-c5like", unet3d_launches(1, 1, 8, (32, 32, 32), encoder_blocks=(1, 2, 2, 4, 4), decoder_blocks=(1, 1, 1, 1, 1))),
        ("golden-nonpow2", unet3d_launches(1, 4, 8, (24, 32, 40))),
    ]
    tr += [("segresnet-" + c.id, _segresnet_case_launches(c)) for c in SC.RELU_CASES + [SC.SMOOTH_CASE, SC.NPOW2_CASE]]
    infer = [("C5", unet3d_launches(3, 1, 48, (128, 128, 128), encoder_blocks=(1, 2, 2, 4, 4), decoder_blocks=(1, 1, 1, 1, 1),
                                    train=False))]
    return tr, infer


def plan_launches():
    tr, infer = plan_launches_by_config()
    for name, launches in tr:
        for split in (False, True):
            for kernel, n, c, dims, view in (l[:5] for l in launches):
                yield name, (kernel, n, c, dims, split, view)
    for name, launches in infer:
        for kernel, n, c, dims, view in (l[:5] for l in launches):
            yield name, (kernel, n, c, dims, False, view)


def plan_gn_bwd_variants():
    """{k_gn_bwd variant: [config, ...]} over the training plans above (the regime key does not carry the variant)"""
    out = {}
    for name, launches in plan_launches_by_config()[0]:
        for l in launches:
            if l[0] == "gn" and l[5] is not None and name not in out.setdefault(l[5], []):
                out[l[5]].append(name)
    return out


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
