"""SegResNet on the GPU (oracle/segresnet_oracle.py: PARITY UNPINNED, MONAI is absent): split-precision logits, sigmoid Dice and every
parameter gradient against fp64, a smooth network held to the noise-floor bounds of tests/segresnet_cases.py, the bf16 mode, the
forward-only, input-gradient, deterministic and CUDA-graph plan kinds, the fused up-sample + skip-add kernel element by element,
and the conv route of every SegResNet convolution."""
import zlib

import pytest
import torch

import segresnet_cases as S
from oracle import sliding_window_inference
from oracle.segresnet_oracle import segresnet_forward
from test_gpu_bandwidth_kernels import check_upsample_skip_add

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _model(pkg, case, precision="split", **kw):
    m = pkg.SegResNet(precision=precision, **case.kw, **kw).to(DEV)
    sd, x, t, scale = S.inputs(case)
    m.load_state_dict(sd, strict=True)
    m.train()
    if scale is not None:
        m.set_dropout_scale(scale.to(DEV))
    return m, x.to(DEV), t.to(DEV)


def _step(pkg, m, x, t):
    out = m(x)
    loss = pkg.DiceLoss(sigmoid=True)(out, t)
    loss.backward()
    return out.detach(), loss.detach()


@pytest.mark.parametrize("case", S.RELU_CASES, ids=lambda c: c.id)
def test_segresnet_split_precision_matches_oracle(pkg, case):
    ref = S.reference(case)
    m, x, t = _model(pkg, case)
    out, loss = _step(pkg, m, x, t)
    b = S.RELU_BOUNDS
    assert S.rel_l2(out, ref["logits"]) < b["logits"]
    assert abs(float(loss) - float(ref["loss"])) < b["loss"] * abs(float(ref["loss"]))
    for k, p in m.named_parameters():
        r = ref[k]
        gn, rn = float(p.grad.double().norm()), float(r.norm())
        assert abs(gn - rn) < b["grad_norm"] * rn + 1e-12, (k, gn, rn)
        cos = float((p.grad.double().cpu() * r).sum() / (gn * rn + 1e-30))
        assert cos > (b["cos_small"] if p.numel() <= 64 else b["cos"]), (k, cos)
    # the forward-only plan (no_grad, eval: no dropout) equals the training plan's forward on the same input
    m.set_dropout_scale(torch.ones(case.shape[0], m.init_filters, device=DEV))
    out_train = m(x).detach()
    m.eval()
    with torch.no_grad():
        out_inf = m(x)
    assert S.rel_l2(out_inf, out_train) < 1e-6      # the same kernels; only the order of the fp64 statistics atomics differs


@pytest.mark.parametrize("input_grad", [False, True])
def test_segresnet_smooth_network_tight_bounds(pkg, input_grad):
    """slope 1 through the public kwargs: every op is smooth, so the split plan is held to the noise-floor bounds"""
    case = S.SMOOTH_CASE
    ref = S.reference(case, input_grad=True)
    m, x, t = _model(pkg, case)
    x.requires_grad_(input_grad)
    out, loss = _step(pkg, m, x, t)
    b = S.SMOOTH_BOUNDS
    assert S.rel_l2(out, ref["logits"]) < b["logits"]
    assert S.rel_l2(loss.reshape(1), ref["loss"]) < b["logits"]
    worst = max((S.rel_l2(p.grad, ref[k]), k) for k, p in m.named_parameters())
    assert worst[0] < b["grad"], worst
    if input_grad:
        assert S.rel_l2(x.grad, ref["dx"]) < b["grad"]


def _check_bf16_dice_bound(pkg, case):
    ref = S.reference(case)
    m, x, t = _model(pkg, case, precision="bf16")
    out, loss = _step(pkg, m, x, t)
    assert abs(float(loss) - float(ref["loss"])) < S.BF16_DICE
    assert S.rel_l2(out, ref["logits"]) < S.BF16_LOGITS
    assert all(torch.isfinite(p.grad).all() for p in m.parameters())


def test_segresnet_bf16_mode_dice_bound(pkg):
    _check_bf16_dice_bound(pkg, S.RELU_CASES[1])


def test_segresnet_npow2_widths_bf16_mode_dice_bound(pkg):
    """widths 24 .. 192, 3 channels per group, 12 input channels, 5 outputs, a forced dropout scale"""
    _check_bf16_dice_bound(pkg, S.NPOW2_CASE)


def test_segresnet_input_gradient_matches_oracle(pkg):
    case = S.RELU_CASES[1]
    ref = S.reference(case, input_grad=True)
    m, x, t = _model(pkg, case)
    x.requires_grad_(True)
    _step(pkg, m, x, t)
    assert S.rel_l2(x.grad, ref["dx"]) < 1e-2
    cos = float((x.grad.double().cpu() * ref["dx"]).sum() / (x.grad.double().norm() * ref["dx"].norm()))
    assert cos > 0.9999


def test_segresnet_deterministic_gradients_bit_identical(pkg):
    case = S.RELU_CASES[1]
    m, x, t = _model(pkg, case, precision="bf16", deterministic=True)
    grads = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        _step(pkg, m, x, t)
        grads.append([p.grad.clone() for p in m.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*grads))


def test_segresnet_graphed_step_equals_eager(pkg):
    case = S.RELU_CASES[1]
    m, x, t = _model(pkg, case, precision="bf16", deterministic=True)
    crit = pkg.DiceLoss(sigmoid=True)
    m.zero_grad(set_to_none=True)
    loss = crit(m(x), t)
    loss.backward()
    loss_e = float(loss)
    del loss                  # no autograd graph of an eager step may be alive when the step is captured
    g_eager = [p.grad.clone() for p in m.parameters()]
    opt = torch.optim.SGD(m.parameters(), lr=0.0)
    step = pkg.train.GraphedTrainStep(m, crit, opt, tuple(x.shape), tuple(t.shape))
    for _ in range(3):
        loss_g = step(x, t)
    torch.cuda.synchronize()
    assert abs(float(loss_g) - loss_e) < 1e-5
    num = sum(float((a.double() - p.grad.double()).pow(2).sum()) for a, p in zip(g_eager, m.parameters())) ** 0.5
    den = sum(float(a.double().pow(2).sum()) for a in g_eager) ** 0.5
    assert num / den < 1e-4


def test_segresnet_sliding_window_inference(pkg):
    """the on-device inferer over a SegResNet vs the oracle inferer driving the fp64 oracle on the host"""
    case = S.RELU_CASES[0]
    m, _, _ = _model(pkg, case)
    m.eval()
    vol = torch.randn(1, 1, 48, 40, 40, generator=torch.Generator().manual_seed(11))
    inf = pkg.predict.SlidingWindowInferer(roi_size=(32, 32, 32), sw_batch_size=2, overlap=0.25, mode="gaussian")
    with torch.no_grad():
        got = inf(vol.to(DEV), m).cpu()
        sd64 = {k: v.double() for k, v in S.inputs(case)[0].items()}
        ref = sliding_window_inference(vol.double(), (32, 32, 32), lambda p: segresnet_forward(sd64, p, *case.blocks, case.groups),
                                       overlap=0.25, mode="gaussian")
    assert S.rel_l2(got, torch.as_tensor(ref)) < 1e-3


# ------------------------------------------------------------------------------------------------ fused up-sample + skip-add
@pytest.mark.parametrize("split", [False, True], ids=["bf16", "split"])
@pytest.mark.parametrize("geom", S.upskip_geometries(), ids=lambda g: "n%d-c%d-%s" % (g[0], g[1], "x".join(map(str, g[2]))))
def test_upsample_skip_add_forward_and_statistics(pkg, geom, split):
    """y = trilinear x2 of p + skip and the per-channel (sum, sumsq) of y, at the SegResNet plans' launch geometries (the bounds:
    tests/test_gpu_bandwidth_kernels.py, whose cases cover every regime of these launches)"""
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(geom).encode()))
    check_upsample_skip_add(pkg.lib, *geom, split, gen)


def test_upsample_skip_add_rejects_a_mismatched_addend(pkg):
    L = pkg.lib
    x, y, s = L.Act.empty(1, 2, 2, 2, 16), L.Act.empty(1, 4, 4, 4, 16), L.Act.empty(1, 4, 4, 2, 16)
    with pytest.raises(RuntimeError, match="addend"):
        L.upsample2x_fwd(x, y, add=s)


# ------------------------------------------------------------------------------------------------ conv routes
@pytest.mark.parametrize("precision", ["bf16", "split"])
def test_segresnet_conv_routes(pkg, precision):
    """the kernel every SegResNet convolution of the BraTS recipe runs on (listed in DESIGN.md)"""
    L = pkg.lib
    L.load_library()
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the table is for a 132-SM H100")
    assert S.route_table(L, precision == "split") == S.BRATS_ROUTES[precision]
