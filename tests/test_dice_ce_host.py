"""DiceCELoss without a GPU: the torch-op restatement against MONAI's published cases and hand-derived values, its closed-form
gradient against fp64 autograd, the errors raised before any launch, and the marshalling of the three C-ABI calls; DiceLoss's
marshalling of the same descriptor, and the options its entry points refuse."""
import contextlib
import ctypes as C
import itertools
import math

import pytest
import torch

from dice_ce_oracle import dice_ce_grad, dice_ce_loss

# MONAI tests/test_dice_ce_loss.py and tests/test_dice_loss.py: input [N=2, C=2, 3], target label map [2, 1, 3]
X = torch.tensor([[[1.0, 1.0, 0.0], [0.0, 0.0, 1.0]], [[1.0, 0.0, 1.0], [0.0, 1.0, 0.0]]], dtype=torch.float64)
T = torch.tensor([[[0.0, 0.0, 1.0]], [[0.0, 1.0, 0.0]]], dtype=torch.float64)

# Every voxel has logits (1, 0) or (0, 1) and its label is the channel holding the 1, so
#   CE = -log(e / (e + 1)) = log(1 + e) - 1 = 0.313262 for every voxel, and so for the mean.
CE = math.log1p(math.e) - 1.0
# softmax Dice: sigma = e / (1 + e) on the labelled channel, 1 - sigma on the other.  In both samples channel 0 holds two labelled
# voxels and one unlabelled one, channel 1 the reverse:
#   ch0: I = 2 sigma, P = 2 sigma + (1 - sigma) = 1 + sigma, T = 2  ->  f0 = 1 - (4 sigma + s) / (3 + sigma + s)
#   ch1: I = sigma,   P = sigma + 2 (1 - sigma) = 2 - sigma, T = 1  ->  f1 = 1 - (2 sigma + s) / (3 - sigma + s)
SIG = math.e / (1.0 + math.e)
_S = 1e-5
DICE_SOFTMAX = 1.0 - 0.5 * ((4 * SIG + _S) / (3 + SIG + _S) + (2 * SIG + _S) / (3 - SIG + _S))


def test_oracle_reproduces_monai_dice_ce_first_case():
    # identity activation: the input equals the one-hot target, so the Dice part is exactly 0 and the loss is the CE
    v = float(dice_ce_loss(X, T, to_onehot_y=True))
    assert abs(v - CE) < 1e-6
    assert abs(v - 0.3133) < 1e-4


def test_oracle_hand_derived_values():
    assert abs(DICE_SOFTMAX - 0.285919) < 1e-6
    assert abs(float(dice_ce_loss(X, T, softmax=True, to_onehot_y=True)) - 0.599181) < 1e-6
    assert abs(DICE_SOFTMAX + CE - 0.599181) < 1e-6
    assert abs(float(dice_ce_loss(X, T, softmax=True, to_onehot_y=True, lambda_ce=2.0)) - 0.912443) < 1e-6
    assert abs(DICE_SOFTMAX + 2 * CE - 0.912443) < 1e-6
    # without background and without activation, channel 1 of the input equals its target exactly: Dice 0, the CE stays
    assert abs(float(dice_ce_loss(X, T, include_background=False, to_onehot_y=True)) - 0.313262) < 1e-6


def test_oracle_dice_part_matches_monai_dice_loss_case():
    # MONAI tests/test_dice_loss.py: include_background=False, to_onehot_y=True, smooth_nr = smooth_dr = 0 -> 0.0
    v = dice_ce_loss(X, T, include_background=False, to_onehot_y=True, smooth_nr=0.0, smooth_dr=0.0, lambda_ce=0.0)
    assert float(v) == 0.0


def _case_inputs(c, form, act, seed):
    g = torch.Generator().manual_seed(seed)
    shape = (2, c, 3, 4, 5)
    x = torch.rand(shape, generator=g, dtype=torch.float64) if act is None else 2.0 * torch.randn(shape, generator=g, dtype=torch.float64)
    lab = torch.randint(0, c, (2, 1, 3, 4, 5), generator=g)
    if form == "label_u8":
        if c > 1:
            lab[0, 0, 0, 0, 0] = c + 3                       # out of range: an all-zero target row
        t = lab.to(torch.uint8) if c > 1 else (torch.rand((2, 1, 3, 4, 5), generator=g) > 0.5).to(torch.uint8)
    elif form == "label_i64":
        if c > 1:
            lab[1, 0, 2, 3, 4] = -1
        t = lab if c > 1 else (torch.rand((2, 1, 3, 4, 5), generator=g) > 0.5).long()
    elif form == "onehot_u8":
        t = torch.nn.functional.one_hot(lab[:, 0], c).movedim(-1, 1).to(torch.uint8) if c > 1 else \
            (torch.rand((2, 1, 3, 4, 5), generator=g) > 0.5).to(torch.uint8)
    else:
        t = torch.softmax(torch.randn(shape, generator=g, dtype=torch.float64), dim=1) if c > 1 else \
            torch.rand((2, 1, 3, 4, 5), generator=g, dtype=torch.float64)
    return x, t


FLAGS = ("include_background", "batch", "squared_pred", "jaccard")


@pytest.mark.parametrize("c", [1, 2, 5])
@pytest.mark.parametrize("form", ["label_u8", "label_i64", "onehot_u8", "soft_f32"])
@pytest.mark.parametrize("act", [None, "sigmoid", "softmax"])
def test_closed_form_gradient_matches_fp64_autograd(c, form, act):
    x, t = _case_inputs(c, form, act, seed=7 * c + len(form))
    for bits in itertools.product((False, True), repeat=len(FLAGS)):
        for reduction in ("mean", "sum"):
            kw = dict(zip(FLAGS, bits))
            kw["include_background"] = not kw["include_background"]
            kw.update(reduction=reduction, sigmoid=act == "sigmoid", softmax=act == "softmax", lambda_dice=0.7, lambda_ce=1.3)
            xx = x.clone().requires_grad_(True)
            dice_ce_loss(xx, t, **kw).backward()
            g = dice_ce_grad(x, t, **kw)
            err = float((g - xx.grad).abs().max())
            assert err < 1e-10, (kw, err)


# ------------------------------------------------------------------------------------------------ errors before any launch
@pytest.fixture()
def no_library(pkg, monkeypatch):
    def boom(*_a, **_k):
        raise AssertionError("the library was touched")
    monkeypatch.setattr(pkg.lib, "load_library", boom)
    monkeypatch.setattr(pkg.lib, "_lib", None)


@pytest.mark.parametrize("kw, exc", [
    (dict(sigmoid=True, softmax=True), ValueError),
    (dict(lambda_dice=-0.1), ValueError),
    (dict(lambda_ce=-1.0), ValueError),
    (dict(reduction="none"), ValueError),
    (dict(other_act=torch.tanh), NotImplementedError),
    (dict(weight=torch.ones(3)), NotImplementedError),
    (dict(ce_weight=torch.ones(3)), NotImplementedError),
    (dict(label_smoothing=0.1), NotImplementedError),
])
def test_constructor_errors(pkg, no_library, kw, exc):
    with pytest.raises(exc):
        pkg.DiceCELoss(**kw)


@pytest.mark.parametrize("xs, ts, kw", [
    ((2, 3, 4, 4, 4), (2, 1, 4, 4), dict(to_onehot_y=True)),            # ranks differ
    ((2, 3, 4, 4, 4), (2, 2, 4, 4, 4), dict(to_onehot_y=True)),         # neither 1 nor C target channels
    ((2, 3, 4, 4, 4), (2, 3, 4, 4, 4), dict(to_onehot_y=True)),         # to_onehot_y on a C-channel target
    ((2, 3, 4, 4, 4), (2, 1, 4, 4, 4), dict()),                         # a label map needs to_onehot_y
    ((2, 3, 4, 4, 4), (2, 1, 4, 4, 5), dict(to_onehot_y=True)),         # spatial shapes differ
])
def test_shape_errors(pkg, no_library, xs, ts, kw):
    with pytest.raises(ValueError):
        pkg.DiceCELoss(softmax=True, **kw)(torch.randn(xs), torch.zeros(ts, dtype=torch.uint8))


def test_cpu_tensor_has_no_fallback(pkg, no_library):
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pkg.DiceCELoss(softmax=True, to_onehot_y=True)(torch.randn(2, 3, 4, 4, 4), torch.zeros(2, 1, 4, 4, 4, dtype=torch.uint8))


def test_one_channel_ignores_softmax_and_to_onehot(pkg, no_library):
    """MONAI only warns for these with C == 1: the constructor and the shape checks accept them (the CPU check then refuses)"""
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pkg.DiceCELoss(softmax=True, to_onehot_y=True)(torch.randn(2, 1, 4, 4, 4), torch.zeros(2, 1, 4, 4, 4, dtype=torch.uint8))


# ------------------------------------------------------------------------------------------------ C-ABI marshalling
class _FakeCuda(torch.Tensor):
    is_cuda = True


HOST_ONLY = {"b200unet_version", "b200unet_last_error", "b200unet_dice_ce_scratch_bytes"}


@pytest.fixture()
def stubbed(pkg, monkeypatch):
    L = pkg.lib
    real = L.load_library()
    calls = []

    class Stub:
        pass
    stub = Stub()
    for name, (res, argtypes) in L._SIGS.items():
        if name in HOST_ONLY:
            setattr(stub, name, getattr(real, name))
            continue

        def make(name=name, argtypes=argtypes):
            def f(*args):
                assert len(args) == len(argtypes), "%s: %d arguments, signature has %d" % (name, len(args), len(argtypes))
                for i, (v, t) in enumerate(zip(args, argtypes)):
                    try:
                        t.from_param(v)
                    except Exception as e:  # noqa: BLE001
                        raise AssertionError("%s: argument %d (%r) does not convert to %s: %s" % (name, i, v, t, e))
                calls.append((name, args))
                return 0
            return f
        setattr(stub, name, make())
    monkeypatch.setattr(L, "_lib", stub)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    monkeypatch.setattr(torch.cuda, "device", lambda *_a, **_k: contextlib.nullcontext())
    return calls


@pytest.mark.parametrize("c, tshape, dtype, kind", [
    (4, (2, 1, 6, 5, 7), torch.uint8, 0),
    (4, (2, 1, 6, 5, 7), torch.int64, 1),
    (4, (2, 1, 6, 5, 7), torch.int32, 1),           # other dtypes go through .long()
    (4, (2, 4, 6, 5, 7), torch.uint8, 2),
    (4, (2, 4, 6, 5, 7), torch.bool, 2),
    (4, (2, 4, 6, 5, 7), torch.float32, 3),
    (1, (2, 1, 6, 5, 7), torch.uint8, 2),           # one channel: the uint8 target itself
    (1, (2, 1, 6, 5, 7), torch.int64, 3),
])
def test_dice_ce_calls_marshal(pkg, stubbed, c, tshape, dtype, kind):
    crit = pkg.DiceCELoss(softmax=True, to_onehot_y=tshape[1] == 1, lambda_ce=0.5)
    x = torch.randn(2, c, 6, 5, 7).as_subclass(_FakeCuda).requires_grad_(True)
    t = torch.zeros(tshape, dtype=dtype).as_subclass(_FakeCuda)
    loss = crit(x, t)
    loss.backward()
    names = [n for n, _ in stubbed]
    assert names == ["b200unet_dice_ce_fwd", "b200unet_dice_ce_bwd"]
    for _, args in stubbed:
        desc = args[0]._obj
        assert desc.target_kind == kind and desc.act == 2 and desc.lambda_ce == 0.5 and desc.reduction == 0
        assert args[3:6] == (2, c, 6 * 5 * 7)
    assert x.grad is not None and x.grad.shape == x.shape


def test_scratch_size_depends_on_the_shape_alone(pkg):
    L = pkg.lib
    d = L.dice_ce_desc(act="softmax", target_kind=0)
    a = L.dice_ce_scratch_bytes(d, 2, 104, 128 ** 3)
    assert a == L.dice_ce_scratch_bytes(L.dice_ce_desc(act="sigmoid", target_kind=0, batch=True), 2, 104, 128 ** 3)
    assert a % 8 == 0 and a >= 8 * 2 * 104 * 5
    assert a < 4 * 2 ** 20                                  # a few slots per sample, not per tile
    with pytest.raises(RuntimeError, match="at most 128"):
        L.dice_ce_scratch_bytes(d, 2, 129, 1000)
    with pytest.raises(RuntimeError, match="int64"):
        L.dice_ce_scratch_bytes(L.dice_ce_desc(target_kind=1), 2, 1, 1000)


@pytest.mark.parametrize("dtype, kind", [(torch.uint8, 2), (torch.bool, 2), (torch.float32, 3), (torch.float16, 3)])
@pytest.mark.parametrize("opts, fields", [
    (dict(sigmoid=True), dict(act=1, include_background=1, squared_pred=0, jaccard=0, batch=0, reduction=0,
                              smooth_nr=1e-5, smooth_dr=1e-5)),
    (dict(include_background=False, squared_pred=True, jaccard=True, batch=True, reduction="sum", smooth_nr=0.5, smooth_dr=2.0),
     dict(act=0, include_background=0, squared_pred=1, jaccard=1, batch=1, reduction=1, smooth_nr=0.5, smooth_dr=2.0)),
])
def test_dice_calls_marshal(pkg, stubbed, dtype, kind, opts, fields):
    """DiceLoss passes its options in the Dice + cross-entropy descriptor, with no CE term"""
    x = torch.randn(2, 3, 6, 5, 7).as_subclass(_FakeCuda).requires_grad_(True)
    t = torch.zeros(2, 3, 6, 5, 7).to(dtype).as_subclass(_FakeCuda)
    pkg.DiceLoss(**opts)(x, t).backward()
    assert [n for n, _ in stubbed] == ["b200unet_dice_fwd", "b200unet_dice_bwd"]
    for _, args in stubbed:
        desc = args[0]._obj
        assert desc.target_kind == kind and desc.lambda_ce == 0.0 and desc.lambda_dice == 1.0
        got = {k: getattr(desc, k) for k in fields}
        assert got == pytest.approx(fields, rel=1e-7), got
        assert args[3:6] == (2, 3, 6 * 5 * 7)
    assert x.grad is not None and x.grad.shape == x.shape


@pytest.mark.parametrize("field, value, status", [
    ("act", 2, -2),                     # softmax: E_UNSUPPORTED
    ("target_kind", 0, -2),             # uint8 label map: E_UNSUPPORTED
    ("target_kind", 1, -2),             # int64 label map: E_UNSUPPORTED
    ("lambda_ce", 0.5, -1),             # a CE term: E_INVALID
])
def test_dice_entry_points_reject_what_only_dice_ce_runs(pkg, field, value, status):
    """b200unet_dice_fwd / _bwd refuse the options only b200unet_dice_ce_* implements, before any CUDA call"""
    L = pkg.lib
    lib = L.load_library()
    d = L.dice_ce_desc(act="sigmoid", target_kind=L.DICE_CE_TARGETS["onehot_u8"], lambda_ce=0.0)
    setattr(d, field, value)
    n, c, s = 2, 3, 64
    logits, target = torch.zeros(n, c, s), torch.zeros(n, c, s, dtype=torch.uint8)
    scratch, loss, g, dlogits = torch.zeros(n * c * 5, dtype=torch.float64), torch.zeros(()), torch.ones(()), torch.zeros(n, c, s)
    assert lib.b200unet_dice_fwd(C.byref(d), logits.data_ptr(), target.data_ptr(), n, c, s, scratch.data_ptr(), loss.data_ptr(),
                                 None) == status
    assert lib.b200unet_last_error().decode().startswith("dice: ")
    assert lib.b200unet_dice_bwd(C.byref(d), logits.data_ptr(), target.data_ptr(), n, c, s, scratch.data_ptr(), g.data_ptr(),
                                 dlogits.data_ptr(), None) == status
    assert "b200unet_dice_ce_" in lib.b200unet_last_error().decode()
