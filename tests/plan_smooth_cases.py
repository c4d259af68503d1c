"""Whole-network plan cases on a smooth network, and the fp64 error model that bounds them.

With ReLU (or LeakyReLU 0.01) a perturbation of 2^-17 on the weights flips activations across the kink and moves the
fp64 oracle's own per-tensor gradients by up to 8e-2, so the ReLU plan tests can only hold gradients to a norm within 3 %
and a cosine above 0.999: a plan wiring error of a few percent (a skip gradient scaled by 0.98, a dropout scale on the
wrong block) passes them.  With activation slope 1 the network is smooth -- conv, GroupNorm / InstanceNorm, trilinear
up-sampling or ConvT, the head and sigmoid Dice -- and the gradients can be held about 15-50x tighter.  The kernels take
the slope as a parameter, so slope 1 runs exactly the schedule and kernels of the real networks, with all-ones masks.

``noise_floor`` models the storage of a split (hi + lo bf16) or single bf16 plan pessimistically: it multiplies the
parameters, the input and the output of every conv, norm and interpolation by 1 + eps * N(0, 1) and reports how far the
fp64 results move.  The bounds below are fixed from that floor, never from what a GPU shows; ``test_plan_smooth_host.py``
checks every row against its floor, ``test_gpu_plan_smooth.py`` checks the plans against the bounds."""
import dataclasses
import os
import sys
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

import oracle.dynunet_oracle as DY
import oracle.unet3d_oracle as U
from oracle import UNetConfig, dice_loss, make_state_dict, unet3d_forward
from oracle.dynunet_oracle import dynunet_forward, make_dynunet_state_dict

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from recipe import dropout_mask, golden_inputs  # noqa: E402

# precision -> bounds on the relative L2 error of the logits (and the loss) and of each gradient tensor (and dx); split
# plans also hold every logit and dx element to elem * rms(reference).  floor_eps / floor_div: the noise floor at floor_eps
# must stay at or below bound / floor_div, so the bound leaves room for the plan's own rounding.
BOUNDS = {
    "split": dict(logits=5e-4, grad=2e-3, elem=1e-2, floor_eps=2.0 ** -16, floor_div=4.0),
    "bf16": dict(logits=5e-2, grad=0.15, elem=None, floor_eps=2.0 ** -8, floor_div=1.0),
}
SMOOTH = 1.0           # the activation slope every row runs at
DROPOUT_P = 0.2


@dataclasses.dataclass
class Case:
    id: str
    arch: str                    # "unet3d" (module kwargs of UNet3D) or "dynunet" (in_channels, out_channels, filters)
    kw: dict
    shape: Tuple[int, ...]       # input (N, C, D, H, W)
    precision: str = "split"
    deterministic: bool = False
    input_grad: bool = False
    train: bool = True           # False: eval-only forward with kw["activation"] applied inside the model
    seed: int = 1


_UNET = dict(n_features=4, n_outputs=3, base_width=8)
_C2 = dict(n_features=4, n_outputs=3, base_width=32)
CASES = [
    Case("unet_default", "unet3d", dict(_UNET), (2, 4, 32, 32, 32)),
    Case("unet_convT", "unet3d", dict(_UNET, use_transposed_convolutions=True), (1, 4, 32, 32, 32), seed=2),
    Case("unet_1ch_5lev", "unet3d", dict(n_features=1, n_outputs=1, base_width=8, encoder_blocks=[1, 2, 2, 4, 4]),
         (1, 1, 32, 32, 48), seed=3),
    Case("unet_blocks_212_122", "unet3d", dict(n_features=2, n_outputs=2, base_width=8, encoder_blocks=[2, 1, 2],
                                               decoder_blocks=[1, 2, 2]), (2, 2, 16, 24, 16), seed=4),
    Case("unet_24x32x40", "unet3d", dict(_UNET), (1, 4, 24, 32, 40), seed=5),
    Case("unet_dil3_groups4", "unet3d", dict(n_features=3, n_outputs=2, base_width=8, feature_dilation=3, norm_groups=4,
                                             encoder_blocks=[1, 2, 2]), (1, 3, 16, 16, 24), seed=6),
    Case("unet_dil3_groups16", "unet3d", dict(n_features=4, n_outputs=2, base_width=8, feature_dilation=3, norm_groups=16,
                                              encoder_blocks=[1, 2, 2]), (2, 4, 16, 16, 16), seed=7),
    Case("unet_24out_bw16", "unet3d", dict(n_features=4, n_outputs=24, base_width=16, encoder_blocks=[1, 2, 2]),
         (1, 4, 32, 32, 32), seed=8),
    Case("unet_12in_dx", "unet3d", dict(n_features=12, n_outputs=2, base_width=16), (1, 12, 32, 32, 32), input_grad=True, seed=9),
    Case("unet_16in_dx", "unet3d", dict(n_features=16, n_outputs=2, base_width=16), (1, 16, 32, 32, 32), input_grad=True, seed=10),
    Case("unet_bw32_det", "unet3d", dict(_C2), (2, 4, 32, 32, 32), deterministic=True, seed=11),
    Case("unet_bw32", "unet3d", dict(_C2), (2, 4, 32, 32, 32), seed=11),
    Case("unet_eval_sigmoid", "unet3d", dict(_UNET, activation="sigmoid"), (1, 4, 32, 32, 32), train=False, seed=12),
    Case("unet_eval_softmax", "unet3d", dict(_UNET, activation="softmax"), (2, 4, 24, 32, 40), train=False, seed=13),
    Case("dyn_8_16_24_32", "dynunet", dict(in_channels=4, out_channels=3, filters=[8, 16, 24, 32]), (1, 4, 32, 32, 32), seed=14),
    Case("dyn_16_24_48", "dynunet", dict(in_channels=1, out_channels=2, filters=[16, 24, 48]), (2, 1, 16, 32, 24), seed=15),
    Case("dyn_5lev", "dynunet", dict(in_channels=4, out_channels=3, filters=[8, 16, 24, 32, 48]), (1, 4, 32, 32, 32), seed=16),
    Case("dyn_24out_dx", "dynunet", dict(in_channels=4, out_channels=24, filters=[16, 32, 48]), (1, 4, 32, 32, 32),
         input_grad=True, seed=17),
    Case("unet_default_bf16", "unet3d", dict(_UNET), (2, 4, 32, 32, 32), precision="bf16"),
    Case("unet_bw32_bf16", "unet3d", dict(_C2), (2, 4, 32, 32, 32), precision="bf16", seed=11),
]


def features(case: Case):
    """The plan wiring paths a row reaches, derived from its configuration (build_unet3d / build_dynunet in plan.cu)."""
    f = {case.arch, case.precision}
    n, cin, *dims = case.shape
    if case.arch == "unet3d":
        cfg = UNetConfig(**case.kw)
        enc, dec = list(cfg.encoder_blocks), cfg.dec_blocks()
        widths = cfg.enc_widths()
        if not case.train:
            f.add("eval_" + cfg.activation)
            return f
        f.add("convT" if cfg.use_transposed_convolutions else "trilinear")
        f.add("dropout_scale_in_dskip" if enc[0] == 1 else "dropout_scale_in")   # block (0,0)'s output is the skip iff one block
        if any(b > 1 for b in dec):
            f.add("decoder_multi_block")
        if cin % 8:
            f.add("padded_input")
        if min(d >> (len(enc) - 1) for d in dims) == 2:
            f.add("bottleneck_2")
        if any(d & (d - 1) for d in dims):
            f.add("extents_not_pow2")
        norm_c = [cin] + widths + [2 * w for w in widths[:-1]]
        if any(U._groups(c, cfg.norm_groups) < c for c in norm_c):
            f.add("gn_multi_channel_groups")
        if any(c >= 8 and U._groups(c, cfg.norm_groups) == c for c in norm_c):
            f.add("gn_one_channel_per_group")
        if cfg.feature_dilation != 2:
            f.add("feature_dilation_%d" % cfg.feature_dilation)
        if cfg.n_outputs > 8:
            f.add("tc_head")
        if case.input_grad:
            f.add("dx_identity" if cin == widths[0] else "dx_sample")
        if widths[0] == 32 and widths[-1] == 256:
            f.add("c2_widths_" + ("deterministic" if case.deterministic else "atomic"))
    else:
        L = len(case.kw["filters"])
        f.add("dyn_%dlev" % L)
        if case.kw["out_channels"] > 8:
            f.add("dyn_tc_head")
        if case.input_grad:
            f.add("dyn_dx")
    if n > 1:
        f.add(case.arch + "_batch2")
    return f


REQUIRED_FEATURES = {
    "trilinear", "dropout_scale_in_dskip", "convT", "padded_input", "bottleneck_2", "dropout_scale_in",
    "decoder_multi_block", "extents_not_pow2", "gn_multi_channel_groups", "gn_one_channel_per_group", "feature_dilation_3",
    "tc_head", "dx_sample", "dx_identity", "c2_widths_deterministic", "c2_widths_atomic", "eval_sigmoid", "eval_softmax",
    "unet3d_batch2", "dyn_3lev", "dyn_4lev", "dyn_5lev", "dyn_tc_head", "dyn_dx", "dynunet_batch2", "split", "bf16",
}


def model_of(pkg, case):
    """the module under test at slope 1: UNet3D through a subclass (the product keeps the reference's ReLU), DynUNet
    through its own act_name"""
    if case.arch == "unet3d":
        class SmoothUNet3D(pkg.UNet3D):
            def _net_desc(self, n, d, h, w):
                nd = super()._net_desc(n, d, h, w)
                nd.act_slope = SMOOTH
                return nd
        return SmoothUNet3D(precision=case.precision, deterministic=case.deterministic, **case.kw)
    L = len(case.kw["filters"])
    return pkg.DynUNet(spatial_dims=3, kernel_size=[[3, 3, 3]] * L, strides=[[1, 1, 1]] + [[2, 2, 2]] * (L - 1),
                       upsample_kernel_size=[[2, 2, 2]] * (L - 1), act_name=("leakyrelu", {"negative_slope": SMOOTH}),
                       precision=case.precision, deterministic=case.deterministic, **case.kw)


# ------------------------------------------------------------------------------------------------ inputs and the oracle
def inputs(case: Case):
    """(fp32 state dict under the module's keys, input, uint8 Dice target, (N, C0) dropout scale or None)"""
    if case.arch == "unet3d":
        cfg = UNetConfig(**case.kw)
        sd = make_state_dict(cfg, seed=case.seed)
        n_out = cfg.n_outputs
    else:
        sd = make_dynunet_state_dict(case.kw["in_channels"], case.kw["out_channels"], case.kw["filters"], seed=case.seed)
        n_out = case.kw["out_channels"]
    x, t, g3 = golden_inputs(case.shape, n_out, seed=case.seed)
    mask = None
    if case.arch == "unet3d" and case.train:
        n, c0 = case.shape[0], cfg.enc_widths()[0]
        mask = dropout_mask(n, c0, DROPOUT_P, g3)
        mask[torch.arange(n), torch.arange(n) % c0] = 0.0     # every sample drops at least one channel
    return sd, x, t, mask


def oracle_forward(case: Case, sd, x, mask, slope):
    if case.arch == "unet3d":
        return unet3d_forward(sd, x, UNetConfig(**case.kw), dropout_mask=mask, slope=slope)
    return dynunet_forward(sd, x, len(case.kw["filters"]), slope)


def reference(case: Case, slope: float = SMOOTH, eps: float = 0.0, noise_seed: int = 0) -> Dict[str, torch.Tensor]:
    """fp64 autograd of the oracle: "logits" (after the model's activation on eval rows), and on training rows "loss" (sigmoid
    Dice), every parameter gradient by state-dict key and, where the row asks for it, "dx".  eps > 0 perturbs as the module
    docstring says."""
    sd, x, t, mask = inputs(case)
    gen = torch.Generator().manual_seed(noise_seed)

    def noisy(v):
        return v * (1 + eps * torch.randn(v.shape, generator=gen, dtype=torch.float64)) if eps else v
    p = {k: noisy(v.double()).requires_grad_(case.train) for k, v in sd.items()}
    xx = noisy(x.double()).requires_grad_(case.input_grad)

    class NoisyF:
        def __getattr__(self, name):
            fn = getattr(F, name)
            if name not in ("conv3d", "conv_transpose3d", "group_norm", "instance_norm", "interpolate"):
                return fn
            return lambda *a, **k: noisy(fn(*a, **k))
    saved = U.F, DY.F
    U.F = DY.F = NoisyF()
    try:
        with torch.set_grad_enabled(case.train):
            out = oracle_forward(case, p, xx, mask, slope)
            res = {"logits": out.detach()}
            if case.train:
                loss = dice_loss(out, t)
                loss.backward()
                res["loss"] = loss.detach().reshape(1)
                res.update({k: v.grad for k, v in p.items()})
                if case.input_grad:
                    res["dx"] = xx.grad
    finally:
        U.F, DY.F = saved
    return res


def rel_l2(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


def bound_of(name: str, precision: str) -> float:
    b = BOUNDS[precision]
    return b["logits"] if name in ("logits", "loss") else b["grad"]


_CACHE: Dict[tuple, Dict[str, torch.Tensor]] = {}


def _cached_reference(case: Case, slope: float, eps: float, noise_seed: int):
    key = (case.arch, repr(sorted(case.kw.items())), case.shape, case.train, case.input_grad, case.seed, slope, eps, noise_seed)
    if key not in _CACHE:
        _CACHE[key] = reference(case, slope, eps, noise_seed)
    return _CACHE[key]


def noise_floor(case: Case, eps: float, slope: float = SMOOTH, runs: int = 2) -> Dict[str, float]:
    """largest relative L2 change of each compared tensor over ``runs`` perturbed fp64 passes"""
    ref = _cached_reference(case, slope, 0.0, 0)
    worst = {k: 0.0 for k in ref}
    for s in range(runs):
        got = _cached_reference(case, slope, eps, s + 1)
        for k in ref:
            worst[k] = max(worst[k], rel_l2(got[k], ref[k]))
    return worst


def real_slope(case: Case) -> float:
    """the activation the architecture actually trains with: the reference UNet3D's ReLU, DynUNet's LeakyReLU(0.01)"""
    return 0.0 if case.arch == "unet3d" else 0.01


def clean_reference(case: Case) -> Dict[str, torch.Tensor]:
    return _cached_reference(case, SMOOTH, 0.0, 0)


def first(arch: str, precision: str = "split") -> Optional[Case]:
    return next((c for c in CASES if c.arch == arch and c.precision == precision and c.train), None)
