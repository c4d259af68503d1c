"""SegResNet plan cases, the fp64 reference they are held to, the noise floor that fixes their bounds, and the conv routes.

``noise_floor`` follows tests/plan_smooth_cases.py: it multiplies the parameters, the input and the output of every conv, norm and
interpolation of the fp64 oracle by 1 + eps * N(0, 1) and reports how far the results move.  The split-precision bounds of the
GPU tests are fixed from that floor on the host (tests/test_segresnet_host.py), never from what a GPU shows."""
import dataclasses
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

import oracle.segresnet_oracle as SR
from oracle import dice_loss
from oracle.segresnet_oracle import make_segresnet_state_dict, segresnet_forward

# split plans on a ReLU network: the bars of the UNet3D / DynUNet plan tests (a 2^-17 perturbation flips activations across the
# kink, so gradients hold a 3 % norm and a 0.999 cosine); on the smooth network (slope 1) the tight split bounds of
# plan_smooth_cases.BOUNDS, which must sit at least floor_div above the noise floor at floor_eps
RELU_BOUNDS = dict(logits=1e-3, loss=1e-3, grad_norm=3e-2, cos=0.999, cos_small=0.995)
SMOOTH_BOUNDS = dict(logits=5e-4, grad=2e-3, floor_eps=2.0 ** -16, floor_div=4.0)
BF16_DICE = 1e-3        # |Dice(plan) - Dice(fp64)| in bf16 mode (test_dynunet_bf16_mode_dice_bound)
BF16_LOGITS = 5e-2


@dataclasses.dataclass
class Case:
    id: str
    kw: dict                      # SegResNet kwargs (MONAI's names)
    shape: Tuple[int, ...]        # input (N, C, D, H, W)
    dropout: bool = False         # a forced Dropout3d scale (kw must set dropout_prob)
    seed: int = 1

    @property
    def groups(self):
        """as MONAI reads them: num_groups counts only with the legacy norm_name spelling; otherwise the norm's kwargs do"""
        if self.kw.get("norm_name"):
            return self.kw.get("num_groups", 8)
        norm = self.kw.get("norm", ("GROUP", {"num_groups": 8}))
        return self.kw.get("num_groups", 8) if isinstance(norm, str) else norm[1].get("num_groups", 8)

    @property
    def blocks(self):
        return tuple(self.kw.get("blocks_down", (1, 2, 2, 4))), tuple(self.kw.get("blocks_up", (1, 1, 1)))


MONAI_DEFAULTS = dict()
BRATS = dict(init_filters=16, in_channels=4, out_channels=3, dropout_prob=0.2, blocks_down=[1, 2, 2, 4], blocks_up=[1, 1, 1])
THREE_LEVEL = dict(in_channels=2, out_channels=24, blocks_down=(2, 1, 2), blocks_up=(1, 2), norm_name="group", num_groups=4)
# widths 24 .. 192 (3 to 24 chunks of 8 channels: no shuffle pattern), 3 channels per group, 12 input channels packed into two
# 8-channel chunks, and level extents down to 3 x 5 x 4
NPOW2 = dict(init_filters=24, in_channels=12, out_channels=5, dropout_prob=0.2, norm=("GROUP", {"num_groups": 8}))
RELU_CASES = [
    Case("monai_defaults", MONAI_DEFAULTS, (1, 1, 32, 32, 32), seed=1),
    Case("brats_recipe", BRATS, (2, 4, 32, 32, 48), dropout=True, seed=2),
    Case("three_level_24out", THREE_LEVEL, (1, 2, 24, 32, 40), seed=3),
    Case("npow2_f24_in12", NPOW2, (2, 12, 24, 40, 32), dropout=True, seed=5),
]
NPOW2_CASE = RELU_CASES[3]
SMOOTH_CASE = Case("smooth_brats_dx", dict(BRATS, init_filters=8, act=("leakyrelu", {"negative_slope": 1.0})), (2, 4, 32, 32, 32),
                   dropout=True, seed=4)


def spec_kw(kw):
    """the oracle's spec arguments of a SegResNet kwargs dict"""
    return dict(in_channels=kw.get("in_channels", 1), out_channels=kw.get("out_channels", 2), init_filters=kw.get("init_filters", 8),
                blocks_down=tuple(kw.get("blocks_down", (1, 2, 2, 4))), blocks_up=tuple(kw.get("blocks_up", (1, 1, 1))))


def slope_of(kw):
    act = kw.get("act", "relu")
    return float(act[1].get("negative_slope", 0.01)) if not isinstance(act, str) and act[0].lower() == "leakyrelu" else 0.0


def inputs(case: Case):
    """(fp32 state dict, input, uint8 Dice target, (N, init_filters) dropout scale or None)"""
    sd = make_segresnet_state_dict(seed=case.seed, **spec_kw(case.kw))
    g = torch.Generator().manual_seed(100 + case.seed)
    x = torch.randn(case.shape, generator=g)
    n_out = case.kw.get("out_channels", 2)
    t = (torch.rand((case.shape[0], n_out) + case.shape[2:], generator=g) > 0.7).to(torch.uint8)
    scale = None
    if case.dropout:
        p = case.kw["dropout_prob"]
        n, f = case.shape[0], case.kw.get("init_filters", 8)
        keep = (torch.rand((n, f), generator=g) >= p).float()
        keep[torch.arange(n), torch.arange(n) % f] = 0.0        # every sample drops at least one channel
        scale = keep / (1.0 - p)
    return sd, x, t, scale


def reference(case: Case, eps: float = 0.0, noise_seed: int = 0, input_grad: bool = False) -> Dict[str, torch.Tensor]:
    """fp64 autograd of the oracle: "logits", "loss" (sigmoid Dice), every parameter gradient by key and, if asked, "dx";
    eps > 0 perturbs as the module docstring says"""
    sd, x, t, scale = inputs(case)
    gen = torch.Generator().manual_seed(noise_seed)

    def noisy(v):
        return v * (1 + eps * torch.randn(v.shape, generator=gen, dtype=torch.float64)) if eps else v
    p = {k: noisy(v.double()).requires_grad_(True) for k, v in sd.items()}
    xx = noisy(x.double()).requires_grad_(input_grad)

    class NoisyF:
        def __getattr__(self, name):
            fn = getattr(F, name)
            if name not in ("conv3d", "group_norm", "interpolate"):
                return fn
            return lambda *a, **k: noisy(fn(*a, **k))
    saved = SR.F
    SR.F = NoisyF()
    try:
        bd, bu = case.blocks
        out = segresnet_forward(p, xx, bd, bu, case.groups, scale, slope_of(case.kw))
        loss = dice_loss(out, t)
        loss.backward()
    finally:
        SR.F = saved
    res = {"logits": out.detach(), "loss": loss.detach().reshape(1)}
    res.update({k: v.grad for k, v in p.items()})
    if input_grad:
        res["dx"] = xx.grad
    return res


def rel_l2(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


def noise_floor(case: Case, eps: float, runs: int = 2, input_grad: bool = True) -> Dict[str, float]:
    """largest relative L2 change of each compared tensor over ``runs`` perturbed fp64 passes"""
    ref = reference(case, input_grad=input_grad)
    worst = {k: 0.0 for k in ref}
    for s in range(runs):
        got = reference(case, eps, s + 1, input_grad=input_grad)
        for k in ref:
            worst[k] = max(worst[k], rel_l2(got[k], ref[k]))
    return worst


# ------------------------------------------------------------------------------------------------ conv routes
def _brats_table(kernels, route, fields):
    """{label: fields of route(launch)} over the BraTS recipe's convolutions of the given kernels (tests/plan_launches.py:
    brats-segresnet).  A label is the layer's state-dict name, with ".dgrad" for a data gradient; the ResBlock convolutions of a
    level share one, "ResBlock L<level>", and must take the same route."""
    import plan_launches as P
    out = {}
    for l in P.BY_NAME["brats-segresnet"].launches():
        if l.kernel in kernels:
            name = l.key[:-len(".conv.weight")]
            if name.endswith((".conv1", ".conv2")):
                name = "ResBlock L%d" % ((l.co // BRATS["init_filters"]).bit_length() - 1)
            r = route(l)
            label, r = name + (".dgrad" if l.kernel == "dgrad" else ""), None if r is None else tuple(r[f] for f in fields)
            assert out.setdefault(label, r) == r, (label, out[label], r)
    return out


# the routes of the BraTS recipe (batch 1, 4 x 224 x 224 x 144, init_filters 16) on a 132-SM H100, (kind, BN, KC) per precision
BRATS_ROUTES = {
    "bf16": {
        "convInit": ("halo", 16, 16), "convInit.dgrad": ("halo", 16, 16),
        "ResBlock L0": ("halo", 16, 16), "ResBlock L0.dgrad": ("halo", 16, 16),
        "ResBlock L1": ("halo", 32, 32), "ResBlock L1.dgrad": ("halo", 32, 32),
        "down_layers.1.0": ("tap", 32, 16), "down_layers.1.0.dgrad": ("class1", 16, 32),
        "ResBlock L2": ("halo", 64, 64), "ResBlock L2.dgrad": ("halo", 64, 64),
        "down_layers.2.0": ("tap", 64, 32), "down_layers.2.0.dgrad": ("class1", 32, 64),
        "ResBlock L3": ("tap", 128, 64), "ResBlock L3.dgrad": ("tap", 128, 64),
        "down_layers.3.0": ("tap", 128, 64), "down_layers.3.0.dgrad": ("class1", 64, 64),
        "up_samples.2.0": ("tap", 16, 32), "up_samples.2.0.dgrad": ("tap", 32, 16),
        "up_samples.1.0": ("tap", 32, 64), "up_samples.1.0.dgrad": ("tap", 64, 32),
        "up_samples.0.0": ("tap", 64, 64), "up_samples.0.0.dgrad": ("tap", 128, 64),
    },
}
BRATS_ROUTES["split"] = {k: (("tap" if v[0] == "halo" else v[0]),) + v[1:] for k, v in BRATS_ROUTES["bf16"].items()}


def route_table(L, split):
    """{label: (kind, BN, KC)} from the library's route query (include/b200unet_diag.h)"""
    from plan_launches import conv_route
    return _brats_table(("fwd", "dgrad"), lambda l: conv_route(L, l, split), ("kind", "bn", "kc"))


# the weight-gradient routes of the BraTS recipe (batch 1, 4 x 224 x 224 x 144, init_filters 16) on a 132-SM H100: (kind, K
# chunk, BN) per precision
BRATS_WGRAD_ROUTES = {
    "bf16": {
        "convInit": ("halo", 64, 16), "ResBlock L0": ("halo", 64, 16), "ResBlock L1": ("halo", 64, 32),
        "down_layers.1.0": ("tap", 16, 32), "ResBlock L2": ("halo", 64, 64), "down_layers.2.0": ("tap", 32, 64),
        "ResBlock L3": ("tap", 64, 128), "down_layers.3.0": ("tap", 64, 128),
        "up_samples.2.0": ("tap", 32, 16), "up_samples.1.0": ("tap", 64, 32), "up_samples.0.0": ("tap", 64, 64),
    },
    "split": {   # no halo mode for hi + lo operands: the per-tap kernel, K chunks of the input width
        "convInit": ("tap", 16, 16), "ResBlock L0": ("tap", 16, 16), "ResBlock L1": ("tap", 32, 32),
        "down_layers.1.0": ("tap", 16, 32), "ResBlock L2": ("tap", 64, 64), "down_layers.2.0": ("tap", 32, 64),
        "ResBlock L3": ("tap", 64, 128), "down_layers.3.0": ("tap", 64, 128),
        "up_samples.2.0": ("tap", 32, 16), "up_samples.1.0": ("tap", 64, 32), "up_samples.0.0": ("tap", 64, 64),
    },
}


def wgrad_route_table(L, split):
    """{label: (kind, K chunk, BN)} from the library's weight-gradient route query"""
    from plan_launches import wgrad_route
    return _brats_table(("wgrad",), lambda l: wgrad_route(L, l, split), ("kind", "cb", "bn"))


# ------------------------------------------------------------------------------------------------ fused up-sampling kernel
def upskip_geometries():
    """(n, C, low-resolution extents) of every up-sample + skip launch of the SegResNet configurations of tests/plan_launches.py"""
    import plan_launches as P
    out = []
    for c in P.CONFIGS:
        for l in c.launches():
            if l.kernel == "up_add" and (l.n, l.c, l.dims) not in out:
                out.append((l.n, l.c, l.dims))
    return out
