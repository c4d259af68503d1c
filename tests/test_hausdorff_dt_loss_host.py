"""HausdorffDTLoss and LogHausdorffDTLoss without a GPU: the scipy restatement of MONAI's distance field against a brute-force
all-pairs field, a hand-derived loss, MONAI's argument defaults, the rejections raised before any launch, the descriptor the
criterion fills and the scratch sizes of the distance-field pass."""
import ctypes as C
import inspect

import numpy as np
import pytest
import torch

from hausdorff_dt_oracle import brute_field, hausdorff_dt_loss, mask_field

CLASSES = ("HausdorffDTLoss", "LogHausdorffDTLoss")


def _masks():
    rng = np.random.default_rng(3)
    out = [rng.random((6, 7, 5)) < q for q in (0.05, 0.3, 0.5, 0.8, 0.97)]
    single = np.zeros((6, 7, 5), dtype=bool)
    single[2, 3, 1] = True
    return out + [single, ~single, np.zeros((6, 7, 5), dtype=bool), np.ones((6, 7, 5), dtype=bool)]


@pytest.mark.parametrize("i", range(9))
def test_oracle_field_is_the_brute_force_field(i):
    m = _masks()[i]
    f = mask_field(m)
    assert f.dtype == np.float32
    assert np.array_equal(f, brute_field(m))
    if m.any() and not m.all():
        assert (f >= 1.0).all()                  # every voxel is at least one step from the other value
    else:
        assert not f.any()


def test_oracle_known_answer():
    """W = 3: p = (0.9, 0.1, 0.1), t = (1, 1, 0) -> pdt = (1, 1, 2), tdt = (2, 1, 1), w = (5, 2, 5) at alpha 2,
    f = (0.01 * 5 + 0.81 * 2 + 0.01 * 5) / 3"""
    p = torch.tensor([0.9, 0.1, 0.1], dtype=torch.float64).reshape(1, 1, 1, 1, 3)
    t = torch.tensor([1.0, 1.0, 0.0], dtype=torch.float64).reshape(1, 1, 1, 1, 3)
    v = float(hausdorff_dt_loss(p, t))
    assert abs(v - 1.72 / 3) < 1e-12
    assert abs(float(hausdorff_dt_loss(p, t, alpha=1.0)) - (0.01 * 3 + 0.81 * 2 + 0.01 * 3) / 3) < 1e-12
    assert abs(float(hausdorff_dt_loss(p, t, log=True)) - np.log(1 + 1.72 / 3)) < 1e-12


@pytest.mark.parametrize("cls", CLASSES)
def test_defaults_match_monai(pkg, cls):
    sig = inspect.signature(getattr(pkg, cls).__init__)
    defaults = {k: v.default for k, v in sig.parameters.items() if k != "self"}
    assert defaults == dict(alpha=2.0, include_background=False, to_onehot_y=False, sigmoid=False, softmax=False, other_act=None,
                            reduction="mean", batch=False)


@pytest.mark.parametrize("cls", CLASSES)
def test_constructor_rejections(pkg, cls):
    L = getattr(pkg, cls)
    with pytest.raises(NotImplementedError, match="other_act"):
        L(other_act=torch.tanh)
    for alpha in (0.0, -1.0):
        with pytest.raises(NotImplementedError, match="alpha"):
            L(alpha=alpha)
    with pytest.raises(ValueError, match="reduction"):
        L(reduction="none")
    with pytest.raises(ValueError):
        L(sigmoid=True, softmax=True)


@pytest.mark.parametrize("cls", CLASSES)
@pytest.mark.parametrize("shape", [(2, 3, 16, 16), (1, 2, 257, 4, 4), (1, 2, 4, 300, 4), (1, 2, 4, 4, 1000), (2, 3, 4, 4, 4, 4)])
def test_shapes_are_rejected_before_any_launch(pkg, cls, shape):
    """2-D (and other) ranks and extents over 256 raise NotImplementedError on CPU tensors: nothing reaches the device"""
    x = torch.zeros(shape)
    t = torch.zeros(shape, dtype=torch.uint8)
    with pytest.raises(NotImplementedError):
        getattr(pkg, cls)(sigmoid=True)(x, t)


def _desc(pkg, **kw):
    opts = dict(act="sigmoid", target_kind=pkg.lib.DICE_CE_TARGETS["onehot_u8"], include_background=False, lambda_dice=0.0,
                voxel_term="hausdorff_dt")
    opts.update(kw)
    return pkg.lib.dice_ce_desc(**opts)


def test_criterion_descriptor(pkg):
    crit = pkg.HausdorffDTLoss(softmax=True, include_background=True, batch=True, reduction="sum", alpha=1.5)
    assert crit.alpha == 1.5 and crit._opts["voxel_term"] == "hausdorff_dt"
    d = pkg.lib.dice_ce_desc(target_kind=0, **crit._opts)
    assert (d.act, d.include_background, d.batch, d.reduction, d.lambda_dice, d.lambda_ce, d.voxel_term) == (2, 1, 1, 1, 0.0, 1.0, 2)
    assert d.hdt_weight is None
    w = torch.zeros(4)
    assert _desc(pkg, hdt_weight=w).hdt_weight == w.data_ptr()
    assert pkg.lib.dice_ce_desc(act="softmax").hdt_weight is None          # DiceCELoss's descriptor leaves the tail zeroed


def test_distance_term_runs_alone(pkg):
    """the loss kernels take the distance-weighted term without a Dice part only"""
    L = pkg.lib
    assert L.dice_ce_scratch_bytes(_desc(pkg), 2, 3, 4096) > 0
    with pytest.raises(RuntimeError, match="distance-weighted"):
        L.dice_ce_scratch_bytes(_desc(pkg, lambda_dice=1.0), 2, 3, 4096)


@pytest.mark.parametrize("n, c, d, h, w, kw", [
    (1, 2, 257, 4, 4, {}), (1, 2, 4, 257, 4, {}), (1, 2, 4, 4, 257, {}), (0, 2, 4, 4, 4, {}), (1, 2, 0, 4, 4, {}),
    (4097, 2, 4, 4, 4, {}), (2, 129, 4, 4, 4, {}), (1, 1, 4, 4, 4, dict(target_kind=1)),
])
def test_scratch_size_is_zero_for_rejected_shapes(pkg, n, c, d, h, w, kw):
    lib = pkg.lib.load_library()
    assert lib.b200unet_hausdorff_dt_scratch_bytes(C.byref(_desc(pkg, **kw)), n, c, d, h, w) == 0
    assert lib.b200unet_last_error().decode().startswith("hausdorff_dt: ")
    with pytest.raises(RuntimeError, match="rejected"):
        pkg.lib.hausdorff_dt_scratch_bytes(_desc(pkg, **kw), n, c, d, h, w)


def test_scratch_size_of_accepted_shapes(pkg):
    """24 bytes per kept (n, c) and voxel (two W-offset and two H-pass planes per mask) plus the foreground counts"""
    L = pkg.lib
    for ib, kept in ((False, 2), (True, 3)):
        b = L.hausdorff_dt_scratch_bytes(_desc(pkg, include_background=ib), 2, 3, 256, 17, 9)
        planes = 24 * 2 * kept * 256 * 17 * 9
        assert planes < b <= planes + 3 * 256
    assert L.hausdorff_dt_scratch_bytes(_desc(pkg), 4096, 2, 1, 1, 1) > 0
    assert L.hausdorff_dt_scratch_bytes(_desc(pkg), 1, 1, 256, 256, 256) > 0   # one channel: include_background is ignored


def test_exported_from_the_package(pkg):
    assert pkg.HausdorffDTLoss is pkg.losses.HausdorffDTLoss
    assert issubclass(pkg.LogHausdorffDTLoss, pkg.HausdorffDTLoss)
