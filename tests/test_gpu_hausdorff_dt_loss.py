"""HausdorffDTLoss and LogHausdorffDTLoss on the GPU: the device distance fields against scipy bit for bit, the loss and dlogits
against fp64 autograd of the restatement (tests/hausdorff_dt_oracle.py), run-to-run bit equality, and a UNet3D training step
whose CUDA graph replays the eager loss."""
import numpy as np
import pytest
import torch
from scipy.ndimage import gaussian_filter

from hausdorff_dt_oracle import activate, distance_fields, hausdorff_dt_loss, kept
from dice_ce_oracle import dice_ce_target
from oracle import UNetConfig, make_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
MARGIN = 1e-4


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


def _blobs(shape, seed, sigma=1.5):
    """smooth random fields of unit spread: thresholded, they are blobs rather than voxel noise"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(shape)
    x = gaussian_filter(x, sigma=(0, 0) + (sigma,) * (len(shape) - 2))
    return torch.from_numpy(x / (x.std() + 1e-12)).float()


def _with_margin(x, sigmoid, softmax):
    """nudge the logits until every activated probability (fp64) is at least MARGIN from 0.5, so fp32 and fp64 masks agree"""
    x = x.clone()
    for _ in range(50):
        p = activate(x.double(), sigmoid, softmax)
        close = (p - 0.5).abs() < 4 * MARGIN
        if not bool(close.any()):
            break
        x[close] += 0.02
    p = activate(x.double(), sigmoid, softmax)
    assert float((p - 0.5).abs().min()) >= MARGIN
    return x


def _inputs(n, c, spatial, act, form, seed):
    """(logits, target as the criterion takes it); form: label_u8, label_i64 (out-of-range labels included), onehot_u8, soft_f32"""
    sigmoid, softmax = act == "sigmoid", act == "softmax"
    shape = (n, c) + tuple(spatial)
    if act is None:                                  # identity: probabilities, as MONAI's tests feed them
        x = torch.sigmoid(2.0 * _blobs(shape, seed))
    else:
        x = 2.0 * _blobs(shape, seed)
    x = _with_margin(x, sigmoid, softmax)
    g = torch.Generator().manual_seed(seed + 1)
    blob = _blobs((n, 1) + tuple(spatial), seed + 2)
    lab = ((blob - blob.min()) / (blob.max() - blob.min() + 1e-12) * c).long().clamp(0, c - 1)
    if form.startswith("label") and c > 1:
        lab[torch.rand(lab.shape, generator=g) < 0.05] = c + 2 if form == "label_u8" else -1
        return x, lab.to(torch.uint8 if form == "label_u8" else torch.int64)
    onehot = dice_ce_target(x.double(), lab) if c > 1 else (blob > 0).double()
    if form == "soft_f32":
        return x, (0.1 + 0.8 * onehot).float()
    return x, onehot.to(torch.uint8)


# ------------------------------------------------------------------------------------------------ distance fields
def _device_fields(pkg, x, t, act, include_background):
    L = pkg.lib
    c = x.shape[1]
    tt = t
    if c > 1 and t.shape[1] == 1:
        kind = L.DICE_CE_TARGETS["label_u8" if t.dtype == torch.uint8 else "label_i64"]
    else:
        kind = L.DICE_CE_TARGETS["onehot_u8" if t.dtype == torch.uint8 else "soft_f32"]
    desc = L.dice_ce_desc(act=act, target_kind=kind, include_background=include_background, lambda_dice=0.0, voxel_term="hausdorff_dt")
    n, _, d, h, w = x.shape
    k = c - 1 if (not include_background and c > 1) else c
    xd, td = x.to(DEV).contiguous(), tt.to(DEV).contiguous()
    scratch = torch.empty(L.hausdorff_dt_scratch_bytes(desc, n, c, d, h, w), dtype=torch.uint8, device=DEV)
    pf = torch.full((n, k, d, h, w), float("nan"), device=DEV)
    tf = torch.full((n, k, d, h, w), float("nan"), device=DEV)
    L.hausdorff_dt_fields(desc, xd, td, scratch, pf, tf)
    torch.cuda.synchronize()
    return pf.cpu(), tf.cpu()


def _scipy_fields(x, t, act, include_background):
    p = activate(x.double(), act == "sigmoid", act == "softmax")
    tt = dice_ce_target(x.double(), t) if x.shape[1] > 1 and t.shape[1] == 1 else t.float()
    p, tt = kept(p, tt, include_background)
    # soft targets: the mask is t > 0.5 in fp32, as stored
    return distance_fields(p), distance_fields(tt.float())


def _check_fields(pkg, x, t, act, include_background):
    pf, tf = _device_fields(pkg, x, t, act, include_background)
    ps, ts = _scipy_fields(x, t, act, include_background)
    assert torch.equal(pf, ps), float((pf - ps).abs().max())
    assert torch.equal(tf, ts), float((tf - ts).abs().max())
    return pf, tf


def test_fields_of_random_blobs(pkg):
    x, t = _inputs(2, 3, (64, 48, 40), "sigmoid", "onehot_u8", seed=1)
    pf, tf = _check_fields(pkg, x, t, "sigmoid", True)
    assert float(pf.max()) > 3 and float(tf.max()) > 3           # blobs: distances well beyond the nearest neighbours


@pytest.mark.parametrize("act, form", [(None, "soft_f32"), ("sigmoid", "onehot_u8")])
def test_fields_along_a_256_long_axis(pkg, act, form):
    x, t = _inputs(1, 1, (256, 17, 9), act, form, seed=2)
    _check_fields(pkg, x, t, act, True)
    # one foreground voxel at one end: the field grows to the far corner
    t = torch.zeros(1, 1, 256, 17, 9, dtype=torch.uint8)
    t[0, 0, 0, 0, 0] = 1
    _, tf = _check_fields(pkg, x, t, act, True)
    assert float(tf.max()) == float(np.float32(np.sqrt(255 ** 2 + 16 ** 2 + 8 ** 2)))


def test_fields_of_a_single_voxel(pkg):
    x = torch.full((1, 2, 9, 10, 11), -3.0)
    x[0, 1, 4, 5, 6] = 3.0
    t = torch.zeros(1, 2, 9, 10, 11, dtype=torch.uint8)
    t[0, 1, 0, 9, 3] = 1
    pf, tf = _check_fields(pkg, x, t, "sigmoid", True)
    assert float(pf[0, 1, 4, 5, 6]) == 1.0 and float(pf[0, 1, 0, 0, 0]) == float(np.float32(np.sqrt(16 + 25 + 36)))
    assert not pf[0, 0].any() and not tf[0, 0].any()                  # channel 0: empty masks
    # a one-voxel volume is either empty or full: the field is 0
    for v in (-1.0, 1.0):
        pf, tf = _check_fields(pkg, torch.full((2, 1, 1, 1, 1), v), torch.ones(2, 1, 1, 1, 1, dtype=torch.uint8), "sigmoid", True)
        assert not pf.any() and not tf.any()


def test_fields_of_empty_and_full_masks_are_zero(pkg):
    x, t = _inputs(2, 3, (12, 10, 9), "sigmoid", "onehot_u8", seed=4)
    x[0, 0], x[1, 1], x[1, 2] = -2.0, 2.0, -2.0
    t[0, 1], t[1, 0], t[1, 2] = 1, 0, 1
    pf, tf = _check_fields(pkg, x, t, "sigmoid", True)
    for f, nc in ((pf, (0, 0)), (pf, (1, 1)), (pf, (1, 2)), (tf, (0, 1)), (tf, (1, 0)), (tf, (1, 2))):
        assert not f[nc].any()
    assert pf[0, 1].any() and tf[0, 0].any()


@pytest.mark.parametrize("form", ["label_u8", "label_i64"])
@pytest.mark.parametrize("include_background", [True, False])
def test_fields_of_label_maps_with_out_of_range_labels(pkg, form, include_background):
    x, t = _inputs(2, 4, (20, 18, 16), "softmax", form, seed=5)
    assert bool(((t < 0) | (t >= 4)).any())
    _check_fields(pkg, x, t, "softmax", include_background)


def test_fields_of_soft_targets_near_one_half(pkg):
    x, _ = _inputs(2, 2, (16, 14, 12), None, "soft_f32", seed=6)
    g = torch.Generator().manual_seed(7)
    t = 0.5 + (torch.randint(-3, 4, x.shape, generator=g).float() * 1e-7)     # 0.5 exactly and its fp32 neighbours
    t[0, 0, :4] = torch.tensor(0.5).nextafter(torch.tensor(1.0))
    assert bool((t == 0.5).any()) and bool((t > 0.5).any()) and bool((t < 0.5).any())
    _check_fields(pkg, x, t, None, True)


# ------------------------------------------------------------------------------------------------ loss and gradient
CASES = [
    # (class, c, act, form, kwargs)
    ("HausdorffDTLoss", 3, "sigmoid", "onehot_u8", dict()),
    ("HausdorffDTLoss", 3, "softmax", "label_u8", dict(include_background=True, reduction="sum")),
    ("HausdorffDTLoss", 1, None, "soft_f32", dict(alpha=1.0)),
    ("HausdorffDTLoss", 1, "sigmoid", "onehot_u8", dict(alpha=2.5, reduction="sum")),
    ("HausdorffDTLoss", 1, "softmax", "soft_f32", dict(include_background=True)),
    ("HausdorffDTLoss", 16, "softmax", "label_i64", dict(batch=True, alpha=2.5)),
    ("HausdorffDTLoss", 16, "sigmoid", "soft_f32", dict(batch=True, reduction="sum", include_background=True)),
    ("HausdorffDTLoss", 16, "softmax", "onehot_u8", dict(alpha=1.0)),
    ("HausdorffDTLoss", 3, "softmax", "onehot_u8", dict(batch=True, reduction="sum", alpha=1.0)),
    ("HausdorffDTLoss", 3, None, "label_i64", dict()),
    ("HausdorffDTLoss", 3, "sigmoid", "label_u8", dict(batch=True, include_background=True, alpha=2.5)),
    ("LogHausdorffDTLoss", 3, "softmax", "label_u8", dict()),
    ("LogHausdorffDTLoss", 1, "sigmoid", "soft_f32", dict(reduction="sum", batch=True)),
]


@pytest.mark.parametrize("i", range(len(CASES)))
def test_loss_and_dlogits_match_fp64_oracle(pkg, i):
    crit, c, act, form, kw = CASES[i]
    x, t = _inputs(2, c, (14, 12, 10), act, form, seed=20 + i)
    akw = dict(sigmoid=act == "sigmoid", softmax=act == "softmax")
    onehot_y = c > 1 and t.shape[1] == 1
    xx = x.to(DEV).requires_grad_(True)
    loss = getattr(pkg, crit)(to_onehot_y=onehot_y, **akw, **kw)(xx, t.to(DEV))
    loss.backward()
    xo = x.double().to(DEV).requires_grad_(True)
    ref = hausdorff_dt_loss(xo, t.to(DEV), log=crit == "LogHausdorffDTLoss", **akw, **kw)
    ref.backward()
    v, vo = float(loss.detach()), float(ref.detach())
    assert vo > 0 and abs(v - vo) <= 1e-5 * abs(vo), (v, vo)
    assert _rel(xx.grad, xo.grad) <= 1e-5, _rel(xx.grad, xo.grad)


def test_bit_identical_run_to_run(pkg):
    x, t = _inputs(2, 16, (64, 64, 64), "softmax", "label_u8", seed=40)
    x, t = x.to(DEV), t.to(DEV)
    crit = pkg.HausdorffDTLoss(softmax=True, to_onehot_y=True)
    runs = []
    for _ in range(3):
        xx = x.clone().requires_grad_(True)
        loss = crit(xx, t)
        loss.backward()
        torch.cuda.synchronize()
        runs.append((loss.detach().clone(), xx.grad.clone()))
    for r in runs[1:]:
        assert torch.equal(r[0], runs[0][0]) and torch.equal(r[1], runs[0][1])


def test_graphed_unet3d_step_replays_the_eager_loss(pkg):
    kw = dict(n_features=2, n_outputs=3, base_width=8)
    sd = make_state_dict(UNetConfig(**kw), seed=6)
    model = pkg.UNet3D(precision="split", dropout=0.0, deterministic=True, **kw).to(DEV)
    model.load_state_dict(sd)
    model.train()
    crit = pkg.HausdorffDTLoss(sigmoid=True)
    g = torch.Generator().manual_seed(13)
    x = torch.randn(2, 2, 16, 16, 16, generator=g)
    t = (_blobs((2, 3, 16, 16, 16), 14) > 0.3).to(torch.uint8)
    eager = crit(model(x.to(DEV)), t.to(DEV))
    eager.backward()
    eager_v = float(eager.detach())
    eager_g = [p.grad.detach().clone() for p in model.ordered_parameters()]
    del eager
    model.zero_grad(set_to_none=True)
    opt = torch.optim.SGD(model.parameters(), lr=0.0)
    step = pkg.train.GraphedTrainStep(model, crit, opt, tuple(x.shape), tuple(t.shape), target_dtype=torch.uint8)
    for _ in range(2):
        v = float(step(x.pin_memory(), t.pin_memory()).detach())
        assert eager_v > 0 and abs(v - eager_v) <= 1e-6 * eager_v, (v, eager_v)
        graph_g = [p.grad.detach().clone() for p in model.ordered_parameters()]
        num = sum(float((a - b).double().pow(2).sum()) for a, b in zip(graph_g, eager_g)) ** 0.5
        den = sum(float(b.double().pow(2).sum()) for b in eager_g) ** 0.5
        assert den > 0 and num / den <= 1e-5, num / den
    assert step.graph is not None
