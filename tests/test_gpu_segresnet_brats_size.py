"""SegResNet at the size README benchmarks it on: the BraTS recipe (init_filters 16, 4 -> 3 channels, blocks_down [1, 2, 2, 4],
blocks_up [1, 1, 1], dropout 0.2 through a forced Dropout3d scale) training on one 4 x 224 x 224 x 144 volume, against the oracle
(oracle/segresnet_oracle.py) on the CPU.  At this size the plan runs what the small plan tests of test_gpu_segresnet.py never
reach: clamped GroupNorm, up-sampling and head grids with partial last sweeps, stream-K weight gradients over every SM, the
persistent halo convolutions over thousands of tiles and k_head_dbias over 220 sweeps.  The route of every convolution and
weight gradient is asserted on the way (segresnet_cases.BRATS_ROUTES, BRATS_WGRAD_ROUTES).

The oracle runs in fp64: about 1.8 T multiply-adds of forward and backward, 139 s of torch's CPU convolutions on 8 threads (fp32
would take about 19 s), once per module; the two GPU steps add about a second.  Bounds (those of the north-star test): split
precision logits rel-L2 <= 1e-3 (measured 1.1e-5 on an H100 80GB HBM3 at 700 W), |dDice| <= 1e-3 |Dice| (1.2e-8), every
gradient norm within 3 % (worst 1.8e-4) and cosine > 0.999; bf16 the Dice bound of the SegResNet plan tests (|dDice| 7.8e-5,
logits rel-L2 6.8e-3)."""
import time

import numpy as np
import pytest
import torch

import segresnet_cases as S
from oracle import dice_loss
from oracle.segresnet_oracle import segresnet_forward

pytestmark = pytest.mark.gpu
DEV = "cuda"
CASE = S.Case("brats_size", S.BRATS, (1, 4, 224, 224, 144), dropout=True, seed=7)


@pytest.fixture(scope="module")
def oracle():
    """fp64 CPU forward + sigmoid Dice + backward of the oracle, with the case's Dropout3d scale"""
    sd, x, t, scale = S.inputs(CASE)
    p = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    t0 = time.perf_counter()
    bd, bu = CASE.blocks
    out = segresnet_forward(p, x.double(), bd, bu, CASE.groups, scale.double(), S.slope_of(CASE.kw))
    loss = dice_loss(out, t)
    loss.backward()
    seconds = time.perf_counter() - t0
    grads = {k: v.grad.numpy() for k, v in p.items()}
    print("SegResNet BraTS-size CPU oracle (fp64, %d threads): %.1f s" % (torch.get_num_threads(), seconds))
    res = dict(sd=sd, x=x, t=t, scale=scale, logits=out.detach().numpy(), dice=float(loss.detach()), grads=grads)
    del out, loss, p
    return res


def _routes(pkg, precision):
    L = pkg.lib
    L.load_library()
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the route tables are for a 132-SM H100")
    assert S.route_table(L, precision == "split") == S.BRATS_ROUTES[precision]
    assert S.wgrad_route_table(L, precision == "split") == S.BRATS_WGRAD_ROUTES[precision]


def _ours(pkg, o, precision):
    m = pkg.SegResNet(precision=precision, **CASE.kw).to(DEV)
    m.load_state_dict(o["sd"], strict=True)
    m.train()
    m.set_dropout_scale(o["scale"].to(DEV))
    out = m(o["x"].to(DEV))
    loss = pkg.DiceLoss(sigmoid=True)(out, o["t"].to(DEV))
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.double().cpu().numpy() for k, p in m.named_parameters()}
    res = out.detach().double().cpu().numpy(), float(loss), grads
    del m, out, loss
    torch.cuda.empty_cache()
    return res


def _rel(a, b):
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


def test_brats_size_split_precision_matches_oracle(pkg, oracle):
    _routes(pkg, "split")
    logits, dice, grads = _ours(pkg, oracle, "split")
    b = S.RELU_BOUNDS
    assert _rel(logits, oracle["logits"]) < b["logits"]
    assert abs(dice - oracle["dice"]) < b["loss"] * abs(oracle["dice"])
    assert set(grads) == set(oracle["grads"])
    norm_dev = max(abs(np.linalg.norm(g) / np.linalg.norm(oracle["grads"][k]) - 1) for k, g in grads.items())
    print("split: logits rel-L2 %.3e, |dDice| %.3e, worst gradient norm deviation %.3e"
          % (_rel(logits, oracle["logits"]), abs(dice - oracle["dice"]), norm_dev))
    for k, g in grads.items():
        r = oracle["grads"][k]
        nr = np.linalg.norm(r)
        assert np.isfinite(g).all(), k
        assert abs(np.linalg.norm(g) - nr) < b["grad_norm"] * nr + 1e-12, (k, np.linalg.norm(g), nr)
        cos = float((g * r).sum() / (np.linalg.norm(g) * nr + 1e-30))
        assert cos > b["cos"], (k, cos)


def test_brats_size_bf16_mode_dice_bound(pkg, oracle):
    _routes(pkg, "bf16")
    logits, dice, grads = _ours(pkg, oracle, "bf16")
    print("bf16: logits rel-L2 %.3e, |dDice| %.3e" % (_rel(logits, oracle["logits"]), abs(dice - oracle["dice"])))
    assert abs(dice - oracle["dice"]) < S.BF16_DICE
    assert all(np.isfinite(g).all() for g in grads.values())
