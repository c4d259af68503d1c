"""FocalLoss, DiceFocalLoss, TverskyLoss and GeneralizedDiceLoss without a GPU: the torch-op restatement
(tests/seg_losses_oracle.py) against closed-form identities and hand-derived values, the kernels' closed-form gradients against
fp64 autograd of it, the errors raised before any launch, the marshalling of every new descriptor field, and the DiceLoss entry
points' refusal of the new options."""
import ctypes as C
import itertools
import math
import warnings

import pytest
import torch
import torch.nn.functional as F

from dice_ce_oracle import dice_ce_loss, dice_ce_target
from seg_losses_oracle import (dice_f, dice_focal_loss, focal_loss, fused_grad, generalized_dice_loss, tversky_loss, W_TYPES)
from test_dice_ce_host import T, X, _FakeCuda, _case_inputs, no_library, stubbed  # noqa: F401  (fixtures)

S1 = 1.0 / (1.0 + math.exp(-1.0))         # sigmoid(1)


# ------------------------------------------------------------------------------------------------ closed-form identities
def _rand(c, seed, shape=(2, 3, 4, 5)):
    g = torch.Generator().manual_seed(seed)
    x = 2.0 * torch.randn((shape[0], c) + shape[1:], generator=g, dtype=torch.float64)
    lab = torch.randint(0, c, (shape[0], 1) + shape[1:], generator=g)
    soft = torch.softmax(torch.randn(x.shape, generator=g, dtype=torch.float64), dim=1)
    return x, lab, soft


def test_sigmoid_focal_with_gamma_0_is_bce_with_logits():
    x, _, soft = _rand(4, 1)
    assert abs(float(focal_loss(x, soft, gamma=0.0)) - float(F.binary_cross_entropy_with_logits(x, soft))) < 1e-14


@pytest.mark.parametrize("form", ["label", "soft"])
def test_softmax_focal_with_gamma_0_is_ce_over_the_classes(form):
    c = 5
    x, lab, soft = _rand(c, 2)
    t = lab if form == "label" else soft
    ce = dice_ce_loss(x, t, lambda_dice=0.0)                  # CE mean over N * S voxels
    assert abs(float(focal_loss(x, t, gamma=0.0, use_softmax=True)) - float(ce) / c) < 1e-14


@pytest.mark.parametrize("act", [None, "sigmoid", "softmax"])
@pytest.mark.parametrize("batch", [False, True])
def test_tversky_at_one_half_without_smoothing_is_dice(act, batch):
    x, lab, _ = _rand(4, 3)
    if act is None:
        x = torch.rand(x.shape, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    kw = dict(sigmoid=act == "sigmoid", softmax=act == "softmax", batch=batch, smooth_nr=0.0, smooth_dr=0.0)
    v = tversky_loss(x, lab, alpha=0.5, beta=0.5, include_background=False, **kw)
    d = dice_ce_loss(x, lab, lambda_ce=0.0, include_background=False, **kw)
    assert abs(float(v) - float(d)) < 1e-14


@pytest.mark.parametrize("batch", [False, True])
def test_uniform_generalized_dice_is_dice_pooled_over_classes(batch):
    x, lab, _ = _rand(4, 5)
    p = torch.softmax(x, dim=1)
    t = dice_ce_target(x, lab)
    v = generalized_dice_loss(x, lab, softmax=True, w_type="uniform", batch=batch)
    # pooling the classes: one channel holding every class's voxels
    pooled = dice_f(p.reshape(2, 1, -1), t.reshape(2, 1, -1), batch=batch).mean()
    assert abs(float(v) - float(pooled)) < 1e-14


# ------------------------------------------------------------------------------------------------ hand-derived values
def test_focal_hand_derived_values():
    # sigmoid form, x = 0, t = 1, gamma = 2: l0 = -logsigmoid(0) = log 2, E = exp(2 logsigmoid(0)) = 1/4  ->  log(2) / 4
    one = torch.ones(1, 1, 1, dtype=torch.float64)
    assert abs(float(focal_loss(0 * one, one)) - math.log(2) / 4) < 1e-15
    assert abs(math.log(2) / 4 - 0.1732868) < 1e-7
    # with alpha = 0.25 the element is scaled by t alpha + (1 - t)(1 - alpha) = 0.25
    assert abs(float(focal_loss(0 * one, one, alpha=0.25)) - math.log(2) / 16) < 1e-15
    # softmax form, logits (0, 0), t = (1, 0): ls = -log 2, p = 1/2, -(1/2)^2 (-log 2) = log(2) / 4 on channel 0, averaged over
    # C' = 2 elements  ->  log(2) / 8
    two = torch.zeros(1, 2, 1, dtype=torch.float64)
    assert abs(float(focal_loss(two, torch.tensor([[[1.0], [0.0]]], dtype=torch.float64), use_softmax=True)) - math.log(2) / 8) < 1e-15
    # MONAI's X / T (logits (1, 0) or (0, 1), the label on the 1): softmax form, ls = log sigmoid(1), (1 - sigmoid(1))^2 =
    # 0.0723295, so each voxel adds 0.0723295 * 0.3132617 = 0.0226580 on its labelled channel; 6 voxels over 12 elements
    v = float(focal_loss(X, T, use_softmax=True))
    assert abs(v - 0.5 * (1 - S1) ** 2 * -math.log(S1)) < 1e-12 and abs(v - 0.0113290) < 1e-7
    # sigmoid form on X (the one-hot target equals X): x = t = 1 gives 0.0226580 as above, x = t = 0 gives log(2) / 4; half each
    v = float(focal_loss(X, T))
    assert abs(v - 0.5 * ((1 - S1) ** 2 * -math.log(S1) + math.log(2) / 4)) < 1e-12 and abs(v - 0.0979724) < 1e-7
    # reduction "sum": the per-(n, c) means over the 3 voxels, summed: 12 / 3 = 4 times the mean
    assert abs(float(focal_loss(X, T, reduction="sum")) - 4 * 0.0979724263) < 1e-9


def test_tversky_and_generalized_dice_hand_derived_values():
    # identity activation on X: one-hot(T) == X, so I = P = T and every f is 1 - (I + s) / (I + s) = 0
    assert float(tversky_loss(X, T)) == 0.0 and float(generalized_dice_loss(X, T)) == 0.0
    # sigmoid, alpha 0.3, beta 0.7, no smoothing.  Sample 0 (sample 1 is the same up to a permutation of voxels):
    #   ch0: p = (s, s, 1/2), t = (1, 1, 0): I = 2s, P - I = 1/2, T - I = 2 - 2s -> f0 = 1 - 2s / (2s + 0.15 + 0.7 (2 - 2s))
    #   ch1: p = (1/2, 1/2, s), t = (0, 0, 1): I = s, P - I = 1, T - I = 1 - s   -> f1 = 1 - s / (s + 0.3 + 0.7 (1 - s))
    s = S1
    f0 = 1 - 2 * s / (2 * s + 0.15 + 0.7 * (2 - 2 * s))
    f1 = 1 - s / (s + 0.3 + 0.7 * (1 - s))
    assert abs(float(tversky_loss(X, T, sigmoid=True, alpha=0.3, beta=0.7, smooth_nr=0, smooth_dr=0)) - (f0 + f1) / 2) < 1e-14
    assert abs(f0 - 0.2647635) < 1e-7 and abs(f1 - 0.4004363) < 1e-7 and abs((f0 + f1) / 2 - 0.3325999) < 1e-7
    # generalized Dice, square weights: w0 = 1/T0^2 = 1/4, w1 = 1
    #   A = 2 (2s / 4 + s) = 3s,  B = (2s + 1/2 + 2) / 4 + (1 + s + 1)  ->  f = 1 - 3s / B, the same for both samples
    B = (2 * s + 2.5) / 4 + 2 + s
    assert abs(float(generalized_dice_loss(X, T, sigmoid=True, smooth_nr=0, smooth_dr=0)) - (1 - 3 * s / B)) < 1e-14
    assert abs(B - 3.7215879) < 1e-7 and abs(1 - 3 * s / B - 0.4106882) < 1e-7


def test_generalized_dice_absent_class_takes_the_largest_weight():
    # one sample, 3 classes, 4 voxels; identity activation.  Class 2 is absent (T2 = 0): w2 = inf -> max(w0, w1)
    p = torch.tensor([[[0.7, 0.2, 0.6, 0.1], [0.2, 0.7, 0.3, 0.8], [0.1, 0.1, 0.1, 0.1]]], dtype=torch.float64)
    lab = torch.tensor([[[0, 1, 0, 0]]])
    # T = (3, 1, 0): square weights (1/9, 1, inf -> 1); I = (1.4, 0.7, 0); P = (1.6, 2.0, 0.4)
    A = 2 * (1.4 / 9 + 0.7 + 0.0)
    B = (1.6 + 3) / 9 + (2.0 + 1) + (0.4 + 0) * 1.0
    assert abs(float(generalized_dice_loss(p, lab, smooth_nr=0, smooth_dr=0)) - (1 - A / B)) < 1e-14
    # simple weights (1/3, 1, inf -> 1)
    A = 2 * (1.4 / 3 + 0.7)
    B = 4.6 / 3 + 3.0 + 0.4
    assert abs(float(generalized_dice_loss(p, lab, w_type="simple", smooth_nr=0, smooth_dr=0)) - (1 - A / B)) < 1e-14


def test_dice_focal_is_the_weighted_sum_of_its_terms():
    x, lab, _ = _rand(4, 6)
    for kw in (dict(softmax=True), dict(sigmoid=True), dict(softmax=True, include_background=False, batch=True)):
        ib = kw.get("include_background", True)
        d = dice_ce_loss(x, lab, lambda_ce=0.0, **kw)
        f = focal_loss(x, lab, include_background=ib, use_softmax=kw.get("softmax", False), gamma=1.5)
        v = dice_focal_loss(x, lab, lambda_dice=0.4, lambda_focal=1.7, gamma=1.5, **kw)
        assert abs(float(v) - (0.4 * float(d) + 1.7 * float(f))) < 1e-13


# ------------------------------------------------------------------------------------------------ closed-form gradients
CASES = [
    # (kind, per-case kwargs of fused_grad; the loss is rebuilt from them below)
    ("focal", dict(focal_softmax=False)),
    ("focal", dict(focal_softmax=False, gamma=0.0, focal_alpha=0.3, weight="w")),
    ("focal", dict(focal_softmax=True)),
    ("focal", dict(focal_softmax=True, gamma=0.0, focal_alpha=0.3, weight="w")),
    ("focal", dict(focal_softmax=True, gamma=0.5, focal_alpha=0.7)),
    ("dice_focal", dict(act="softmax")),
    ("dice_focal", dict(act="sigmoid", squared_pred=True, focal_alpha=0.25)),
    ("dice_focal", dict(act=None, jaccard=True, gamma=1.0)),
    ("tversky", dict(alpha=0.3, beta=0.7)),
    ("tversky", dict(alpha=0.8, beta=0.1)),
] + [("gdice", dict(w_type=w)) for w in W_TYPES]


def _loss(kind, x, t, act, ib, batch, reduction, kw):
    sig, smx = act == "sigmoid", act == "softmax"
    common = dict(include_background=ib, reduction=reduction)
    if kind == "focal":
        return focal_loss(x, t, gamma=kw.get("gamma", 2.0), alpha=kw.get("focal_alpha"), weight=kw.get("weight"),
                          use_softmax=kw["focal_softmax"], **common)
    if kind == "dice_focal":
        return dice_focal_loss(x, t, sigmoid=sig, softmax=smx, squared_pred=kw.get("squared_pred", False), jaccard=kw.get("jaccard", False),
                               batch=batch, gamma=kw.get("gamma", 2.0), alpha=kw.get("focal_alpha"), lambda_dice=0.6, lambda_focal=1.4,
                               **common)
    if kind == "tversky":
        return tversky_loss(x, t, sigmoid=sig, softmax=smx, alpha=kw["alpha"], beta=kw["beta"], batch=batch, **common)
    return generalized_dice_loss(x, t, sigmoid=sig, softmax=smx, w_type=kw["w_type"], batch=batch, **common)


def _grad(kind, x, t, act, ib, batch, reduction, kw):
    kw = dict(kw)
    if kind == "focal":
        kw.update(lambda_dice=0.0, lambda_focal=1.0)
        act = None
    elif kind == "dice_focal":
        kw.update(lambda_dice=0.6, lambda_focal=1.4, focal_softmax=act == "softmax")
    else:
        kw.update(kind={"gdice": "gdice"}.get(kind, kind))
    kw["act"] = act
    return fused_grad(x, t, include_background=ib, batch=batch, reduction=reduction, **kw)


@pytest.mark.parametrize("c", [1, 2, 5])
@pytest.mark.parametrize("form", ["label_u8", "label_i64", "onehot_u8", "soft_f32"])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_closed_form_gradient_matches_fp64_autograd(c, form, case):
    kind, kw = CASES[case]
    acts = [kw["act"]] if "act" in kw else ([None] if kind == "focal" else [None, "sigmoid", "softmax"])
    for act in acts:
        x, t = _case_inputs(c, form, "softmax" if act is None and kind == "focal" else act, seed=11 * c + len(form) + case)
        if kind == "gdice" and c > 1 and form != "soft_f32":
            # an absent class in sample 0: its square / simple weight is infinite
            t = t.clone()
            if t.shape[1] == 1:
                t[0][t[0] == c - 1] = 0
            else:
                t[0, c - 1] = 0
        for ib, batch, reduction in itertools.product((True, False), (False, True), ("mean", "sum")):
            kk = dict(kw)
            if kk.get("weight") == "w":
                kept = c - 1 if (not ib and c > 1) else c
                kk["weight"] = torch.linspace(0.5, 2.0, kept, dtype=torch.float64)
            xx = x.clone().requires_grad_(True)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                _loss(kind, xx, t, act, ib, batch, reduction, kk).backward()
            g = _grad(kind, x, t, act, ib, batch, reduction, kk)
            if c - (not ib and c > 1) == 1 and kind == "focal" and kk["focal_softmax"]:
                # a softmax over one channel: ls = 0, p = 1, the loss is 0 for every logit and so is its gradient.  Autograd agrees
                # except where it meets 0 * (1 - p)^(gamma - 1) = 0 * inf (0 < gamma < 1)
                assert bool((g == 0).all()) and bool(((xx.grad == 0) | torch.isnan(xx.grad)).all())
                continue
            err = float((g - xx.grad).abs().max())
            assert err < 1e-10, (kind, kk, act, ib, batch, reduction, err)


# ------------------------------------------------------------------------------------------------ errors before any launch
@pytest.mark.parametrize("cls, kw, exc", [
    ("FocalLoss", dict(reduction="none"), ValueError),
    ("FocalLoss", dict(weight=[1.0, -0.5]), ValueError),
    ("FocalLoss", dict(gamma=-1.0), ValueError),
    ("DiceFocalLoss", dict(sigmoid=True, softmax=True), ValueError),
    ("DiceFocalLoss", dict(lambda_dice=-0.1), ValueError),
    ("DiceFocalLoss", dict(lambda_focal=-1.0), ValueError),
    ("DiceFocalLoss", dict(reduction="none"), ValueError),
    ("DiceFocalLoss", dict(other_act=torch.tanh), NotImplementedError),
    ("DiceFocalLoss", dict(weight=torch.ones(3)), NotImplementedError),
    ("TverskyLoss", dict(sigmoid=True, softmax=True), ValueError),
    ("TverskyLoss", dict(reduction="none"), ValueError),
    ("TverskyLoss", dict(other_act=torch.tanh), NotImplementedError),
    ("GeneralizedDiceLoss", dict(w_type="cubic"), ValueError),
    ("GeneralizedDiceLoss", dict(sigmoid=True, softmax=True), ValueError),
    ("GeneralizedDiceLoss", dict(reduction="batch"), ValueError),
    ("GeneralizedDiceLoss", dict(other_act=torch.tanh), NotImplementedError),
])
def test_constructor_errors(pkg, no_library, cls, kw, exc):
    with pytest.raises(exc):
        getattr(pkg, cls)(**kw)


NEW = ("FocalLoss", "DiceFocalLoss", "TverskyLoss", "GeneralizedDiceLoss")


@pytest.mark.parametrize("cls", NEW)
@pytest.mark.parametrize("xs, ts, kw", [
    ((2, 3, 4, 4, 4), (2, 1, 4, 4), dict(to_onehot_y=True)),            # ranks differ
    ((2, 3, 4, 4, 4), (2, 2, 4, 4, 4), dict(to_onehot_y=True)),         # neither 1 nor C target channels
    ((2, 3, 4, 4, 4), (2, 3, 4, 4, 4), dict(to_onehot_y=True)),         # to_onehot_y on a C-channel target
    ((2, 3, 4, 4, 4), (2, 1, 4, 4, 4), dict()),                         # a label map needs to_onehot_y
    ((2, 3, 4, 4, 4), (2, 1, 4, 4, 5), dict(to_onehot_y=True)),         # spatial shapes differ
])
def test_shape_errors(pkg, no_library, cls, xs, ts, kw):
    with pytest.raises(ValueError):
        getattr(pkg, cls)(**kw)(torch.randn(xs), torch.zeros(ts, dtype=torch.uint8))


@pytest.mark.parametrize("cls", NEW)
def test_cpu_tensor_has_no_fallback(pkg, no_library, cls):
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        getattr(pkg, cls)(to_onehot_y=True)(torch.randn(2, 3, 4, 4, 4), torch.zeros(2, 1, 4, 4, 4, dtype=torch.uint8))


def test_focal_softmax_without_background_ignores_alpha(pkg, no_library):
    with pytest.warns(UserWarning, match="alpha"):
        crit = pkg.FocalLoss(use_softmax=True, include_background=False, alpha=0.25)
    assert crit._opts["focal_alpha"] is None
    with pytest.warns(UserWarning, match="alpha"):
        crit = pkg.DiceFocalLoss(softmax=True, include_background=False, alpha=0.25)
    assert crit._opts["focal_alpha"] is None
    assert pkg.FocalLoss(use_softmax=False, include_background=False, alpha=0.25)._opts["focal_alpha"] == 0.25


def test_exported(pkg):
    from importlib import import_module
    losses = import_module("3dunetcnn_b200.losses")
    for name in NEW:
        assert getattr(pkg, name) is getattr(losses, name)


# ------------------------------------------------------------------------------------------------ C-ABI marshalling
def _marshal(pkg, stubbed, crit, c=4, tshape=(2, 1, 6, 5, 7), dtype=torch.uint8):
    x = torch.randn(2, c, 6, 5, 7).as_subclass(_FakeCuda).requires_grad_(True)
    t = torch.zeros(tshape, dtype=dtype).as_subclass(_FakeCuda)
    crit(x, t).backward()
    assert [n for n, _ in stubbed] == ["b200unet_dice_ce_fwd", "b200unet_dice_ce_bwd"]
    descs = [args[0]._obj for _, args in stubbed]
    for _, args in stubbed:
        assert args[3:6] == (2, c, 6 * 5 * 7)
    assert x.grad is not None and x.grad.shape == x.shape
    return descs


def _fields(desc, fields):
    got = {k: getattr(desc, k) for k in fields}
    assert got == pytest.approx(fields, rel=1e-7), got


BASE = dict(squared_pred=0, jaccard=0, smooth_nr=1e-5, smooth_dr=1e-5)


@pytest.mark.parametrize("opts, fields", [
    (dict(to_onehot_y=True, sigmoid=True, alpha=0.2, beta=0.9, batch=True, reduction="sum"),
     dict(act=1, target_kind=0, include_background=1, batch=1, reduction=1, lambda_dice=1.0, lambda_ce=0.0, overlap=1,
          tversky_alpha=0.2, tversky_beta=0.9, w_type=0, voxel_term=0, focal_use_alpha=0, **BASE)),
    (dict(to_onehot_y=True, softmax=True, include_background=False, smooth_nr=0.0, smooth_dr=1e-3),
     dict(act=2, target_kind=0, include_background=0, batch=0, reduction=0, lambda_dice=1.0, lambda_ce=0.0, overlap=1,
          tversky_alpha=0.5, tversky_beta=0.5, voxel_term=0, squared_pred=0, jaccard=0, smooth_nr=0.0, smooth_dr=1e-3)),
])
def test_tversky_marshal(pkg, stubbed, opts, fields):
    for d in _marshal(pkg, stubbed, pkg.TverskyLoss(**opts)):
        _fields(d, fields)
        assert d.class_weight is None


@pytest.mark.parametrize("w_type, code", [("square", 0), ("simple", 1), ("uniform", 2), ("SIMPLE", 1)])
def test_generalized_dice_marshal(pkg, stubbed, w_type, code):
    crit = pkg.GeneralizedDiceLoss(to_onehot_y=True, softmax=True, w_type=w_type, batch=True)
    for d in _marshal(pkg, stubbed, crit, tshape=(2, 1, 6, 5, 7), dtype=torch.int64):
        _fields(d, dict(act=2, target_kind=1, overlap=2, w_type=code, batch=1, lambda_dice=1.0, lambda_ce=0.0, voxel_term=0, **BASE))


@pytest.mark.parametrize("opts, fields", [
    (dict(), dict(act=0, include_background=1, lambda_dice=0.0, lambda_ce=1.0, voxel_term=1, focal_softmax=0, focal_gamma=2.0,
                  focal_use_alpha=0, overlap=0, reduction=0)),
    (dict(use_softmax=True, gamma=0.5, alpha=0.3, reduction="sum"),
     dict(act=0, lambda_dice=0.0, lambda_ce=1.0, voxel_term=1, focal_softmax=1, focal_gamma=0.5, focal_use_alpha=1,
          focal_alpha=0.3, reduction=1)),
    (dict(include_background=False, gamma=0.0, alpha=0.0),
     dict(include_background=0, voxel_term=1, focal_softmax=0, focal_gamma=0.0, focal_use_alpha=1, focal_alpha=0.0)),
])
def test_focal_marshal(pkg, stubbed, opts, fields):
    for d in _marshal(pkg, stubbed, pkg.FocalLoss(to_onehot_y=True, **opts)):
        _fields(d, fields)
        assert d.class_weight is None


@pytest.mark.parametrize("weight, ib, expect", [
    (0.5, True, [0.5] * 4),
    ([1.0, 2.0, 3.0, 4.0], True, [1.0, 2.0, 3.0, 4.0]),
    (torch.tensor([2.0, 0.0, 1.0]), False, [2.0, 0.0, 1.0]),
])
def test_focal_class_weights_marshal(pkg, stubbed, weight, ib, expect):
    """the weights reach the kernels as one fp32 buffer per device, built on the first call and reused after it"""
    crit = pkg.FocalLoss(to_onehot_y=True, include_background=ib, weight=weight)
    descs = _marshal(pkg, stubbed, crit)
    (w,) = crit._weights.values()
    assert w.dtype == torch.float32 and w.tolist() == pytest.approx(expect)
    for d in descs:
        assert d.class_weight == w.data_ptr() and d.voxel_term == 1 and d.include_background == int(ib)
    stubbed.clear()
    for d in _marshal(pkg, stubbed, crit):
        assert d.class_weight == w.data_ptr()


def test_focal_weight_length_must_match_the_kept_classes(pkg, stubbed):
    with pytest.raises(ValueError, match="number of classes"):
        _marshal(pkg, stubbed, pkg.FocalLoss(to_onehot_y=True, weight=[1.0, 2.0, 3.0]))
    # one kept class: weights are ignored, as in MONAI
    for d in _marshal(pkg, stubbed, pkg.FocalLoss(weight=[1.0, 2.0]), c=1, tshape=(2, 1, 6, 5, 7)):
        assert d.class_weight is None


@pytest.mark.parametrize("opts, fields", [
    (dict(to_onehot_y=True, softmax=True),
     dict(act=2, target_kind=0, include_background=1, lambda_dice=1.0, lambda_ce=1.0, voxel_term=1, focal_softmax=1,
          focal_gamma=2.0, focal_use_alpha=0, overlap=0)),
    (dict(to_onehot_y=True, sigmoid=True, include_background=False, squared_pred=True, jaccard=True, batch=True, reduction="sum",
          gamma=1.5, alpha=0.25, lambda_dice=0.3, lambda_focal=2.0, smooth_nr=0.1, smooth_dr=0.2),
     dict(act=1, include_background=0, squared_pred=1, jaccard=1, batch=1, reduction=1, lambda_dice=0.3, lambda_ce=2.0,
          voxel_term=1, focal_softmax=0, focal_gamma=1.5, focal_use_alpha=1, focal_alpha=0.25, smooth_nr=0.1, smooth_dr=0.2)),
])
def test_dice_focal_marshal(pkg, stubbed, opts, fields):
    for d in _marshal(pkg, stubbed, pkg.DiceFocalLoss(**opts)):
        _fields(d, fields)
        assert d.class_weight is None


@pytest.mark.parametrize("tshape, dtype, kind", [
    ((2, 1, 6, 5, 7), torch.uint8, 0), ((2, 1, 6, 5, 7), torch.int32, 1), ((2, 4, 6, 5, 7), torch.bool, 2),
    ((2, 4, 6, 5, 7), torch.float32, 3),
])
@pytest.mark.parametrize("cls", NEW)
def test_target_forms_marshal(pkg, stubbed, cls, tshape, dtype, kind):
    crit = getattr(pkg, cls)(to_onehot_y=tshape[1] == 1)
    for d in _marshal(pkg, stubbed, crit, tshape=tshape, dtype=dtype):
        assert d.target_kind == kind


def test_descriptor_defaults_are_todays_dice_ce(pkg):
    """a zeroed tail is the Dice overlap with the CE term: DiceCELoss's descriptor leaves it zeroed"""
    d = pkg.lib.dice_ce_desc(act="softmax")
    for k in ("overlap", "tversky_alpha", "tversky_beta", "w_type", "voxel_term", "focal_softmax", "focal_gamma", "focal_alpha",
              "focal_use_alpha"):
        assert getattr(d, k) == 0, k
    assert d.class_weight is None


def test_scratch_bytes_checks_the_new_fields(pkg):
    L = pkg.lib
    d = L.dice_ce_desc(act="softmax", overlap="tversky")
    assert L.dice_ce_scratch_bytes(d, 2, 16, 4096) == L.dice_ce_scratch_bytes(L.dice_ce_desc(act="softmax"), 2, 16, 4096)
    with pytest.raises(RuntimeError, match="squared_pred"):
        L.dice_ce_scratch_bytes(L.dice_ce_desc(act="softmax", overlap="tversky", squared_pred=True), 2, 16, 4096)
    with pytest.raises(RuntimeError, match="focal_gamma"):
        L.dice_ce_scratch_bytes(L.dice_ce_desc(voxel_term="focal", focal_gamma=-1.0), 2, 16, 4096)
    bad = L.dice_ce_desc()
    bad.overlap = 3
    with pytest.raises(RuntimeError, match="overlap"):
        L.dice_ce_scratch_bytes(bad, 2, 16, 4096)


@pytest.mark.parametrize("field, value", [
    ("overlap", 1), ("overlap", 2), ("voxel_term", 1), ("focal_softmax", 1), ("focal_use_alpha", 1), ("class_weight", 64),
])
def test_dice_entry_points_reject_the_new_options(pkg, field, value):
    """b200unet_dice_fwd / _bwd refuse every option only b200unet_dice_ce_* implements with E_UNSUPPORTED, before any CUDA call"""
    L = pkg.lib
    lib = L.load_library()
    d = L.dice_ce_desc(act="sigmoid", target_kind=L.DICE_CE_TARGETS["onehot_u8"], lambda_ce=0.0)
    setattr(d, field, value)
    n, c, s = 2, 3, 64
    logits, target = torch.zeros(n, c, s), torch.zeros(n, c, s, dtype=torch.uint8)
    scratch, loss, g, dlogits = torch.zeros(n * c * 5, dtype=torch.float64), torch.zeros(()), torch.ones(()), torch.zeros(n, c, s)
    assert lib.b200unet_dice_fwd(C.byref(d), logits.data_ptr(), target.data_ptr(), n, c, s, scratch.data_ptr(), loss.data_ptr(),
                                 None) == -2
    assert lib.b200unet_last_error().decode().startswith("dice: ")
    assert lib.b200unet_dice_bwd(C.byref(d), logits.data_ptr(), target.data_ptr(), n, c, s, scratch.data_ptr(), g.data_ptr(),
                                 dlogits.data_ptr(), None) == -2
    assert "b200unet_dice_ce_" in lib.b200unet_last_error().decode()
