"""FocalLoss, DiceFocalLoss, TverskyLoss and GeneralizedDiceLoss on the GPU: every case of tests/seg_loss_cases.py against fp64
autograd of the torch-op restatement (tests/seg_losses_oracle.py), the Dice part left finite at infinite logits when the focal
weight is 0, run-to-run bit equality at 104 classes, and a DynUNet training step whose CUDA graph replays the eager loss."""
import warnings

import pytest
import torch

import seg_loss_cases as S
from oracle.dynunet_oracle import make_dynunet_state_dict
from seg_losses_oracle import dice_focal_loss, focal_loss, generalized_dice_loss, tversky_loss
from test_gpu_dice_ce import _inputs, _rel
from oracle import dice_loss

pytestmark = pytest.mark.gpu
DEV = "cuda"
ORACLES = {"FocalLoss": focal_loss, "DiceFocalLoss": dice_focal_loss, "TverskyLoss": tversky_loss,
           "GeneralizedDiceLoss": generalized_dice_loss}


def _case_inputs(crit, kw, c, form, spatial, seed):
    act = "softmax" if kw.get("softmax") else ("sigmoid" if kw.get("sigmoid") else None)
    # focal terms read raw logits; the identity activation of an overlap reads probabilities as MONAI's tests feed them
    x, t, onehot_y = _inputs(c, form, "sigmoid" if crit == "FocalLoss" else act, spatial, seed)
    if S.absent_class(crit, c, form):
        t = t.clone()
        if t.shape[1] == 1:
            t[0][t[0] == c - 1] = 0
        else:
            t[0, 0] = t[0, 0] | t[0, c - 1]          # the voxels of class c - 1 move to class 0
            t[0, c - 1] = 0
    return x, t, onehot_y


def _resolve(kw, c):
    kw = dict(kw)
    if kw.get("weight") == S.WEIGHTS:
        kept = c - 1 if (not kw.get("include_background", True) and c > 1) else c
        kw["weight"] = torch.linspace(0.5, 2.0, kept).tolist()
    return kw


def _run(pkg, crit, x, t, **kw):
    xx = x.detach().to(DEV).float().requires_grad_(True)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        loss = getattr(pkg, crit)(**kw)(xx, t.to(DEV))
    loss.backward()
    return float(loss.detach()), xx.grad.detach().double().cpu()


def _oracle(crit, x, t, **kw):
    xx = x.detach().double().to(DEV).requires_grad_(True)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        loss = ORACLES[crit](xx, t.to(DEV), **kw)
    loss.backward()
    return float(loss.detach()), xx.grad.detach().cpu()


@pytest.mark.parametrize("form", S.FORMS)
@pytest.mark.parametrize("c", S.CLASSES)
@pytest.mark.parametrize("crit", list(S.VARIANTS))
def test_kernels_match_fp64_oracle_autograd(pkg, crit, c, form):
    spatial = S.spatial_of(c)
    for i, var in enumerate(S.VARIANTS[crit]):
        x, t, onehot_y = _case_inputs(crit, var, c, form, spatial, seed=c * 17 + len(form) * 3 + len(crit) + i)
        kw = dict(_resolve(var, c), to_onehot_y=onehot_y)
        v, g = _run(pkg, crit, x, t, **kw)
        vo, go = _oracle(crit, x, t, **kw)
        assert abs(v - vo) <= 1e-5 * abs(vo) + 1e-7, (crit, kw, v, vo)
        assert _rel(g, go) <= 1e-4, (crit, kw, _rel(g, go))


@pytest.mark.parametrize("c", [1, 3])
def test_dice_part_stays_finite_at_infinite_logits_without_the_focal_term(pkg, c):
    """lambda_focal = 0 evaluates no focal term: a sigmoid saturates at +-inf, so the loss and dlogits equal fp64 DiceLoss"""
    g = torch.Generator().manual_seed(9)
    x = torch.randn(2, c, 5, 6, 7, generator=g)
    x.view(-1)[::7] = float("inf")
    x.view(-1)[3::11] = -float("inf")
    t = (torch.rand(x.shape, generator=g) > 0.5).to(torch.uint8)
    for kw in (dict(), dict(squared_pred=True, batch=True), dict(jaccard=True, reduction="sum")):
        v, gr = _run(pkg, "DiceFocalLoss", x, t, sigmoid=True, lambda_focal=0.0, **kw)
        xr = x.double().requires_grad_(True)
        lr = dice_loss(xr, t, sigmoid=True, **kw)
        lr.backward()
        assert abs(v - float(lr)) <= 1e-5 * abs(float(lr)), (kw, v, float(lr))
        assert bool(torch.isfinite(gr).all()) and _rel(gr, xr.grad) <= 1e-4, kw


def test_gamma_zero_has_no_nan(pkg):
    """(1 - p)^0 is 1 even where p = 1: saturated logits give a finite focal term in both forms"""
    x = torch.zeros(2, 3, 4, 4, 4)
    x[:, 0] = 60.0                                     # softmax p_0 = 1 to fp32 precision
    lab = torch.zeros(2, 1, 4, 4, 4, dtype=torch.uint8)
    for kw in (dict(use_softmax=True), dict()):
        v, g = _run(pkg, "FocalLoss", x, lab, gamma=0.0, to_onehot_y=True, **kw)
        vo, go = _oracle("FocalLoss", x, lab, gamma=0.0, **kw)
        assert torch.isfinite(torch.tensor(v)) and bool(torch.isfinite(g).all())
        assert abs(v - vo) <= 1e-5 * abs(vo) + 1e-7 and float((g - go).abs().max()) < 1e-6


@pytest.mark.parametrize("crit, kw", [
    ("DiceFocalLoss", dict(softmax=True, include_background=False)),
    ("FocalLoss", dict(use_softmax=True)),
    ("TverskyLoss", dict(softmax=True, alpha=0.3, beta=0.7)),
    ("GeneralizedDiceLoss", dict(softmax=True, batch=True)),
])
def test_bit_identical_run_to_run_at_104_classes(pkg, crit, kw):
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 104, 64, 64, 64, generator=g).to(DEV)
    lab = torch.randint(0, 104, (2, 1, 64, 64, 64), generator=g).to(torch.uint8).to(DEV)
    loss_fn = getattr(pkg, crit)(to_onehot_y=True, **kw)
    runs = []
    for _ in range(2):
        xx = x.clone().requires_grad_(True)
        loss = loss_fn(xx, lab)
        loss.backward()
        torch.cuda.synchronize()
        runs.append((loss.detach().clone(), xx.grad.clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_dynunet_16_class_graphed_step_replays_the_eager_dice_focal_loss(pkg):
    kw = dict(spatial_dims=3, in_channels=2, out_channels=16, kernel_size=[[3, 3, 3]] * 3, strides=[[1, 1, 1]] + [[2, 2, 2]] * 2,
              upsample_kernel_size=[[2, 2, 2]] * 2, filters=[16, 24, 32])
    model = pkg.DynUNet(precision="split", **kw).to(DEV)
    model.load_state_dict(make_dynunet_state_dict(2, 16, kw["filters"], seed=4), strict=True)
    model.train()
    crit = pkg.DiceFocalLoss(softmax=True, to_onehot_y=True)
    g = torch.Generator().manual_seed(12)
    x = torch.randn(2, 2, 16, 16, 16, generator=g)
    lab = torch.randint(0, 16, (2, 1, 16, 16, 16), generator=g).to(torch.uint8)
    eager = crit(model(x.to(DEV)), lab.to(DEV))
    eager.backward()
    eager_v = eager.detach().clone()
    del eager
    model.zero_grad(set_to_none=True)
    opt = torch.optim.SGD(model.parameters(), lr=0.0)
    step = pkg.train.GraphedTrainStep(model, crit, opt, tuple(x.shape), tuple(lab.shape), target_dtype=torch.uint8)
    for _ in range(2):
        v = step(x.pin_memory(), lab.pin_memory()).detach().clone()
        assert torch.equal(v, eager_v), (float(v), float(eager_v))
    assert step.graph is not None
