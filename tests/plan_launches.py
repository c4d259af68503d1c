"""The launches of the plan builders of 3dunetcnn_b200/csrc/plan.cu, restated once, and the configurations the host tests derive
their cases from.  ``unet3d``, ``dynunet`` and ``segresnet`` take the module's constructor kwargs, the batch, the input extents
and the plan flags, and return the convolutions and bandwidth-bound kernels (tests/bandwidth_cases.py) of the plan in plan.cu's
emit order.  tests/test_plan_launches_host.py holds every configuration of ``CONFIGS`` to the library's MAC count and parameter
spec; each consumer picks its configurations from ``CONFIGS`` by name."""
import os
import sys
from dataclasses import dataclass
from typing import Optional, Tuple

import bench
import conv_route_cases as R
import segresnet_cases as S

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from recipe import CASES as GOLDEN  # noqa: E402


@dataclass(frozen=True)
class Launch:
    """one launch.  Channel counts are real ones; the view a kernel reads pads them to a multiple of 8 (``pad8``), which only
    the packed network input needs."""
    kernel: str                  # fwd dgrad wgrad gn act_bwd up_fwd up_add up_bwd bias_grad head_fwd head_bwd head_dbias
    key: str                     # state-dict key of the conv or head weight, or the norm's prefix ("" for the others)
    n: int
    c: int                       # channels read: a conv's source (data gradient: the output gradient), a norm's input
    dims: Tuple[int, int, int]   # conv: extents of the output (weight gradient: of dy); up-sampling: of the low-resolution side
    op: str = ""                 # conv: k3s1, k3s2, k1, class1, class2, k2s2 (conv_route_cases.conv_geometry)
    co: int = 0                  # conv: output channels (weight gradient: of dy)
    mode: int = 0                # conv epilogue: 1 = the GroupNorm + activation backward
    key2: str = ""               # conv: weight key and channels of a fused 1x1x1 second source
    c2: int = 0
    reads_input: bool = False    # a data gradient into the packed network input (emit_dgrad's reads_input)
    macs_div: int = 1            # conv_role's macs_div, for a transposed layer launched over its output grid
    view: bool = False           # bandwidth kernels: the up-sampling's full-resolution operand is a channel slice of a concat
    variant: Optional[str] = None   # gn of a training plan: what k_gn_bwd adds and scales ("plain", "add1", "add1+scale")
    lo_out: bool = False         # conv: the output has a lo plane in bf16 plans too (plan.cu: new_buf's force_lo)

    def macs(self):
        """the algorithmic MACs the plan counts for a convolution (plan.cu: conv_macs): on the grid of the layer's output (data
        and weight gradient: of dy), so the parity-class launches over the fine grid count one voxel in eight"""
        div = self.macs_div * (8 if self.op.startswith("class") else 1)
        taps = {"k1": 1, "k2s2": 8, "class2": 8}.get(self.op, 27)
        return self.n * self.dims[0] * self.dims[1] * self.dims[2] * self.co * (self.c * taps + self.c2) // div


def pad8(c):
    return -(-c // 8) * 8


def conv_route(L, l, split):
    """the library's route of a forward or data-gradient launch (conv_route_cases.conv_query)"""
    return R.conv_query(L, l.op, pad8(l.c), pad8(l.co), l.dims, split, l.mode, pad8(l.c2), n=l.n, lo_out=l.lo_out)


def wgrad_route(L, l, split):
    """the library's route of a weight-gradient launch (conv_route_cases.wgrad_query)"""
    return R.wgrad_query(L, l.op, pad8(l.c), pad8(l.co), l.dims, split, n=l.n)


def route_table(L, config, split, label):
    """{label(key) (+ ".dgrad" for a data gradient): (kind, BN, KC, CTAs per SM)} of the config's forward convolutions and
    data gradients, from the library's route query (include/b200unet_diag.h)"""
    return {label(l.key) + (".dgrad" if l.kernel == "dgrad" else ""): tuple(conv_route(L, l, split)[f]
                                                                           for f in ("kind", "bn", "kc", "blocks_per_sm"))
            for l in config.launches() if l.kernel in ("fwd", "dgrad")}


def wgrad_route_table(L, config, split, label):
    """{label(key): (kind, K chunk, BN)} of the config's weight gradients, from the library's weight-gradient route query"""
    return {label(l.key): tuple(wgrad_route(L, l, split)[f] for f in ("kind", "cb", "bn"))
            for l in config.launches() if l.kernel == "wgrad"}


def _block_fwd(out, n, keys, cin, C, e, train, first=False, scale_in=False):
    """build_block_fwd: norm1 -> conv1 -> norm2 -> conv2 + the 1x1x1 `sample` convolution of the input when the width changes.
    build_block_bwd hands norm1's k_gn_bwd the output gradient as the residual addend when the width is kept (and the Dropout3d
    scale when the input is the dropout output); the network's first block runs no k_gn_bwd for norm1."""
    n1, c1, n2, c2, cs = keys
    sample = cin != C
    v1 = None if first or not train else "plain" if sample else "add1+scale" if scale_in else "add1"
    out += [Launch("gn", n1, n, cin, e, variant=v1), Launch("fwd", c1, n, cin, e, "k3s1", C),
            Launch("gn", n2, n, C, e, variant="plain" if train else None),
            Launch("fwd", c2, n, C, e, "k3s1", C, key2=cs if sample else "", c2=cin if sample else 0)]
    return keys, cin, C, e, first


def _block_bwd(out, n, block, input_grad):
    """build_block_bwd: the weight gradients, and the data gradients through the norm + act epilogue; below the network's first
    block only input_grad plans run the sample convolution's"""
    (n1, c1, n2, c2, cs), cin, C, e, first = block
    sample = cin != C
    out.append(Launch("wgrad", c2, n, C, e, "k3s1", C))
    if sample:
        out.append(Launch("wgrad", cs, n, cin, e, "k1", C))
    out += [Launch("dgrad", c2, n, C, e, "k3s1", C, mode=1), Launch("wgrad", c1, n, cin, e, "k3s1", C),
            Launch("dgrad", c1, n, C, e, "k3s1", cin, mode=1, reads_input=first)]
    if sample and (input_grad or not first):
        out.append(Launch("dgrad", cs, n, C, e, "k1", cin, reads_input=first))


def unet3d(n, dims, train=True, input_grad=False, **kw):
    """build_unet3d for UNet3D(**kw): residual blocks (unet3d_block_keys) and a stride-2 convolution below every encoder level;
    per decoder stage its blocks at the width it receives, then the 1x1x1 convolution to the next width and the x2 up-sampling
    into the low half of the concat buffer, or the transposed convolution (LAYER_CONVT_ZI: a 3x3x3 convolution over the
    zero-inserted input, whose backward adds the bias gradient).  The head has no bias."""
    eb = list(kw.get("encoder_blocks") or (1, 2, 2, 4))
    L = len(eb)
    db = list(kw.get("decoder_blocks") or [1] * L)
    W = [kw.get("base_width", 32) << k for k in range(L)]
    ext = [tuple(d >> k for d in dims) for k in range(L)]
    convT = kw.get("use_transposed_convolutions", False)
    out, enc, dec, stages = [], [[] for _ in range(L)], [], []

    def keys(pre, b):
        pre += ".blocks.%d" % b
        return (pre + ".conv1.norm1", pre + ".conv1.conv.weight", pre + ".conv2.norm1", pre + ".conv2.conv.weight",
                pre + ".sample.weight")
    cin = kw.get("n_features", 1)
    for k in range(L):
        for b in range(eb[k]):
            enc[k].append(_block_fwd(out, n, keys("encoder.layers.%d" % k, b), cin, W[k], ext[k], train, first=k == b == 0,
                                     scale_in=(k, b) == (0, 1) and kw.get("dropout", 0.2) > 0))
            cin = W[k]
        if k + 1 < L:
            out.append(Launch("fwd", "encoder.downsampling_convolutions.%d.weight" % k, n, W[k], ext[k + 1], "k3s2", W[k]))
    for i in range(L):
        depth, C = L - 1 - i, (cin if i + 1 < L else W[0])
        dec.append([_block_fwd(out, n, keys("decoder.layers.%d" % i, b), C if b else cin, C, ext[depth], train)
                    for b in range(db[i])])
        if not depth:
            break
        out_w = W[depth - 1]
        if convT:
            key = "decoder.upsampling_blocks.%d.weight" % i
            out.append(Launch("fwd", key, n, cin, ext[depth - 1], "k3s1", out_w, macs_div=8))
        else:
            key = "decoder.pre_upsampling_blocks.%d.weight" % i
            out += [Launch("fwd", key, n, cin, ext[depth], "k1", out_w), Launch("up_fwd", "", n, out_w, ext[depth], view=True)]
        stages.append((key, depth, cin, out_w))
        cin = 2 * out_w
    out.append(Launch("head_fwd", "final_convolution.weight", n, W[0], dims))
    if not train:
        return out
    out.append(Launch("head_bwd", "", n, W[0], dims))
    for blk in reversed(dec[L - 1]):
        _block_bwd(out, n, blk, input_grad)
    for i in range(L - 2, -1, -1):
        key, depth, in_w, out_w = stages[i]
        if convT:
            out += [Launch("bias_grad", "", n, out_w, ext[depth - 1], view=True),
                    Launch("wgrad", key, n, in_w, ext[depth - 1], "k3s1", out_w, macs_div=8),
                    Launch("dgrad", key, n, out_w, ext[depth], "k3s2", in_w)]
        else:
            out += [Launch("up_bwd", "", n, out_w, ext[depth], view=True), Launch("wgrad", key, n, in_w, ext[depth], "k1", out_w),
                    Launch("dgrad", key, n, out_w, ext[depth], "k1", in_w)]
        for blk in reversed(dec[i]):
            _block_bwd(out, n, blk, input_grad)
    for k in range(L - 1, -1, -1):
        for blk in reversed(enc[k]):
            _block_bwd(out, n, blk, input_grad)
        if k:       # emit_down_bwd
            key = "encoder.downsampling_convolutions.%d.weight" % (k - 1)
            out += [Launch("wgrad", key, n, W[k - 1], ext[k], "k3s2", W[k - 1]),
                    Launch("dgrad", key, n, W[k - 1], ext[k - 1], "class1", W[k - 1])]
    return out


def dynunet(n, dims, train=True, input_grad=False, **kw):
    """build_dynunet for DynUNet(**kw) with strides 1, 2, 2, ...: per level a post-activation block (build_dyn_block_fwd: conv1,
    stride 2 below level 0 -> InstanceNorm -> act -> conv2 -> InstanceNorm -> act); per decoder stage the kernel-2 transposed
    convolution (parity class 2) into the low half of the concat buffer and a block reading all of it.  The backward of a block
    (build_dyn_block_bwd) runs act_bwd on its second norm and plain k_gn_bwd on both; conv1's data gradient is parity class 1
    at stride 2.  The head has a bias, whose gradient k_head_dbias computes up to 8 outputs."""
    F = list(kw["filters"])
    L = len(F)
    ext = [tuple(d >> k for d in dims) for k in range(L)]
    out, enc, dec = [], [], [None] * (L - 1)

    def block_fwd(pre, cin, C, k, stride):
        out.extend([Launch("fwd", pre + ".conv1.conv.weight", n, cin, ext[k], "k3s%d" % stride, C),
                    Launch("gn", pre + ".norm1", n, C, ext[k], variant="plain" if train else None),
                    Launch("fwd", pre + ".conv2.conv.weight", n, C, ext[k], "k3s1", C),
                    Launch("gn", pre + ".norm2", n, C, ext[k], variant="plain" if train else None)])
        return pre, cin, C, k, stride

    def block_bwd(block):
        pre, cin, C, k, stride = block
        k1, k2 = pre + ".conv1.conv.weight", pre + ".conv2.conv.weight"
        out.extend([Launch("act_bwd", "", n, C, ext[k]), Launch("wgrad", k2, n, C, ext[k], "k3s1", C),
                    Launch("dgrad", k2, n, C, ext[k], "k3s1", C, mode=1), Launch("wgrad", k1, n, cin, ext[k], "k3s%d" % stride, C)])
        if stride == 2:
            out.append(Launch("dgrad", k1, n, C, ext[k - 1], "class1", cin))
        elif input_grad or pre != "input_block":
            out.append(Launch("dgrad", k1, n, C, ext[k], "k3s1", cin, reads_input=pre == "input_block"))
    for i in range(L):
        name = "input_block" if i == 0 else "bottleneck" if i == L - 1 else "downsamples.%d" % (i - 1)
        enc.append(block_fwd(name, kw.get("in_channels", 1) if i == 0 else F[i - 1], F[i], i, 1 if i == 0 else 2))
    for u in range(L - 1):
        lo, hi = L - 1 - u, L - 2 - u
        out.append(Launch("fwd", "upsamples.%d.transp_conv.conv.weight" % u, n, F[lo], ext[hi], "class2", F[hi]))
        dec[hi] = block_fwd("upsamples.%d.conv_block" % u, 2 * F[hi], F[hi], hi, 1)
    out.append(Launch("head_fwd", "output_block.conv.conv.weight", n, F[0], dims))
    if not train:
        return out
    out.append(Launch("head_bwd", "", n, F[0], dims))
    if kw.get("out_channels", 1) <= 8:
        out.append(Launch("head_dbias", "", n, F[0], dims))
    for hi in range(L - 1):
        block_bwd(dec[hi])
        key = "upsamples.%d.transp_conv.conv.weight" % (L - 2 - hi)
        out += [Launch("wgrad", key, n, F[hi], ext[hi + 1], "k2s2", F[hi + 1]),
                Launch("dgrad", key, n, F[hi], ext[hi + 1], "k2s2", F[hi + 1])]
    for i in range(L - 1, -1, -1):
        block_bwd(enc[i])
    return out


def segresnet(n, dims, train=True, input_grad=False, **kw):
    """build_segresnet for SegResNet(**kw): convInit, per level a stride-2 convolution (below the first) and its ResBlocks (the
    residual blocks at a kept width; the first takes the Dropout3d output when dropout_prob is set); per decoder stage the 1x1x1
    convolution to C channels, the fused x2 up-sampling + skip-add into a whole C-channel buffer (up_add) and its blocks.  The
    head normalises F channels (act_bwd on that norm alone) into the biased 1x1x1 convolution."""
    F = kw.get("init_filters", 8)
    bd, bu = list(kw.get("blocks_down", (1, 2, 2, 4))), list(kw.get("blocks_up", (1, 1, 1)))
    L = len(bd)
    W = [F << k for k in range(L)]
    ext = [tuple(d >> k for d in dims) for k in range(L)]
    nin = kw.get("in_channels", 1)
    out, enc, dec = [], [[] for _ in range(L)], [[] for _ in range(L - 1)]

    def keys(pre):
        return pre + ".norm1", pre + ".conv1.conv.weight", pre + ".norm2", pre + ".conv2.conv.weight", ""
    out.append(Launch("fwd", "convInit.conv.weight", n, nin, ext[0], "k3s1", F))
    for i in range(L):
        if i:
            out.append(Launch("fwd", "down_layers.%d.0.conv.weight" % i, n, W[i - 1], ext[i], "k3s2", W[i]))
        for b in range(bd[i]):
            enc[i].append(_block_fwd(out, n, keys("down_layers.%d.%d" % (i, b + 1)), W[i], W[i], ext[i], train,
                                     scale_in=i == b == 0 and (kw.get("dropout_prob") or 0) > 0))
    for i in range(L - 1):
        j = L - 2 - i
        out += [Launch("fwd", "up_samples.%d.0.conv.weight" % i, n, 2 * W[j], ext[j + 1], "k1", W[j]),
                Launch("up_add", "", n, W[j], ext[j + 1])]
        for b in range(bu[i]):
            dec[i].append(_block_fwd(out, n, keys("up_layers.%d.%d" % (i, b)), W[j], W[j], ext[j], train))
    out += [Launch("gn", "conv_final.0", n, F, dims, variant="plain" if train else None),
            Launch("head_fwd", "conv_final.2.conv.weight", n, F, dims)]
    if not train:
        return out
    out.append(Launch("head_bwd", "", n, F, dims))
    if kw.get("out_channels", 2) <= 8:
        out.append(Launch("head_dbias", "", n, F, dims))
    out.append(Launch("act_bwd", "", n, F, dims))
    for i in range(L - 2, -1, -1):
        j = L - 2 - i
        for blk in reversed(dec[i]):
            _block_bwd(out, n, blk, input_grad)
        key = "up_samples.%d.0.conv.weight" % i
        out += [Launch("up_bwd", "", n, W[j], ext[j + 1]), Launch("wgrad", key, n, 2 * W[j], ext[j + 1], "k1", W[j]),
                Launch("dgrad", key, n, W[j], ext[j + 1], "k1", 2 * W[j])]
    for i in range(L - 1, -1, -1):
        for blk in reversed(enc[i]):
            _block_bwd(out, n, blk, input_grad)
        if i:       # emit_down_bwd
            key = "down_layers.%d.0.conv.weight" % i
            out += [Launch("wgrad", key, n, W[i - 1], ext[i], "k3s2", W[i]),
                    Launch("dgrad", key, n, W[i], ext[i - 1], "class1", W[i - 1])]
    out.append(Launch("wgrad", "convInit.conv.weight", n, nin, ext[0], "k3s1", F))
    if input_grad:
        out.append(Launch("dgrad", "convInit.conv.weight", n, F, ext[0], "k3s1", nin, reads_input=True))
    return out


# ------------------------------------------------------------------------------------------------------ configurations
@dataclass(frozen=True)
class Config:
    name: str
    arch: str                    # the module: "UNet3D", "DynUNet" or "SegResNet"
    kw: dict                     # its constructor kwargs
    n: int
    dims: Tuple[int, int, int]
    train: bool = True           # False: a forward-only plan
    input_grad: bool = False     # the plan also computes the gradient of the input

    def launches(self):
        return {"UNet3D": unet3d, "DynUNet": dynunet, "SegResNet": segresnet}[self.arch](self.n, self.dims, self.train,
                                                                                          self.input_grad, **self.kw)


def _bench(name, config=None, **kw):
    c = bench.CONFIGS[name]
    if c["kind"] == "train":
        return Config(config or name, "UNet3D", dict(c["model"], **kw), c["batch"], tuple(c["volume"]))
    return Config(config or name, "UNet3D", dict(c["model"], **kw), c["sw_batch"], tuple(c["roi"]), train=False)


# examples/brats2020/brats2020_config.json: filters 64 .. 384 over six levels, 128^3 patches
BRATS_DYNUNET = dict(in_channels=4, out_channels=3, kernel_size=[[3, 3, 3]] * 6, strides=[[1, 1, 1]] + [[2, 2, 2]] * 5,
                     upsample_kernel_size=[[2, 2, 2]] * 5, filters=[64, 96, 128, 192, 256, 384])
# the benchmark's C2 (also with transposed convolutions), C3 and C5 (the forward of one sw_batch of roi tiles); the BraTS DynUNet
# (batch 2) and SegResNet recipe: training at 1 x 224 x 224 x 144 and 2 x 128^3, the two shapes tools/segresnet_bench.py times,
# and its forward-only plan; the golden recipes of tests/golden/recipe.py and the SegResNet plan cases of tests/segresnet_cases.py
CONFIGS = [_bench("C2"), _bench("C2", "C2-convT", use_transposed_convolutions=True), _bench("C3"), _bench("C5"),
           Config("brats-dynunet", "DynUNet", BRATS_DYNUNET, 2, (128, 128, 128)),
           Config("brats-segresnet", "SegResNet", S.BRATS, 1, (224, 224, 144), input_grad=True),
           Config("brats-segresnet-128", "SegResNet", S.BRATS, 2, (128, 128, 128)),
           Config("brats-segresnet-infer", "SegResNet", S.BRATS, 1, (224, 224, 144), train=False)]
CONFIGS += [Config("golden-" + name, "UNet3D", kw, shape[0], tuple(shape[2:])) for name, (kw, shape) in GOLDEN.items()]
CONFIGS += [Config("segresnet-" + c.id, "SegResNet", c.kw, c.shape[0], tuple(c.shape[2:]), input_grad=True)
            for c in S.RELU_CASES + [S.SMOOTH_CASE]]
BY_NAME = {c.name: c for c in CONFIGS}
