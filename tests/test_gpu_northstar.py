"""Parity at the size BASELINE.json's north_star states it on: 4-channel 128^3 volumes, UNet3D base_width=32
(reference unet3d/models/pytorch/segmentation/unet.py:47-50 driven as training_utils.py:101-112), against the CPU
fp32 oracle ("the reference's own nn.Conv3d forward/backward").  At this size every production dispatch is active:
halo mode of the convolution kernel in bf16 (inputs of <= 64 channels), per-tap tiles for wider inputs (128->128@64^3,
256->256@32^3), in split precision and on the 16^3 level, the weight-gradient kernel.  C3 at the size bench.py measures it
(160 x 192 x 128: more tiles per persistent halo CTA, other stream-K weight-gradient splits, 20 x 24 x 16 at the bottleneck) and a
C3-shaped crop (80 x 96 x 64: non-cubic tile walks, 10 x 12 x 8 at the bottleneck) are held to the same bars.  C3 at full size,
measured on an H100 80GB HBM3 at 700 W: split logits rel-L2 9.9e-6, |dDice| 6.0e-8, worst gradient norm deviation 3.5e-4; bf16
logits 4.9e-3, |dDice| 1.2e-5, whole gradient 5.6e-3, worst norm deviation 5.3e-3.  Its fp32 CPU oracle takes 30 s (C2: 17 s).

Tolerances (north_star): logits rel-L2 <= 1e-3 and |dDice| <= 1e-3 in `split` precision; every gradient norm within
3 % and cosine > 0.999.  In single-pass `bf16` the Dice bound holds and the logits carry bf16 operand rounding
(<= 2e-2, measured 4.9e-3), the whole gradient vector is within 3e-2 rel-L2 of the fp64-pinned oracle's (measured
5.6e-3 / 6.7e-3) and every gradient norm within 5 % (measured <= 5.7e-3); per-tensor bounds against torch's own bf16
autocast are in test_gpu_bf16_vs_autocast.py."""
import os

import numpy as np
import pytest
import torch

from oracle import UNetConfig, make_state_dict, unet3d_forward, dice_loss

pytestmark = pytest.mark.gpu
DEV = "cuda"
KW = dict(n_features=4, n_outputs=3, base_width=32)


def _inputs(shape, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g, dtype=torch.float32)
    t = (torch.rand((shape[0], KW["n_outputs"]) + tuple(shape[2:]), generator=torch.Generator().manual_seed(seed + 1)) > 0.7).to(torch.uint8)
    return x, t


def _oracle(shape, seed):
    """fp32 CPU oracle forward + Dice + backward (dropout mask = identity)."""
    cfg = UNetConfig(**KW)
    sd = make_state_dict(cfg, seed=0)
    x, t = _inputs(shape, seed)
    sdr = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref = unet3d_forward(sdr, x, cfg)
    loss = dice_loss(ref, t)
    loss.backward()
    grads = {k: v.grad.double().numpy() for k, v in sdr.items()}
    return dict(sd=sd, x=x, t=t, logits=ref.detach().double().numpy(), dice=float(loss), grads=grads)


@pytest.fixture(scope="module")
def oracle_c2():
    return _oracle((1, 4, 128, 128, 128), seed=21)


@pytest.fixture(scope="module")
def oracle_c3():
    return _oracle((1, 4, 160, 192, 128), seed=41)


@pytest.fixture(scope="module")
def oracle_c3crop():
    return _oracle((1, 4, 80, 96, 64), seed=31)


def _ours(pkg, o, precision):
    model = pkg.UNet3D(precision=precision, **KW).to(DEV)
    model.load_state_dict(o["sd"], strict=True)
    model.train()
    model.set_dropout_scale(torch.ones(o["x"].shape[0], KW["base_width"]))
    out = model(o["x"].to(DEV))
    loss = pkg.DiceLoss(sigmoid=True)(out, o["t"].to(DEV))
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.double().cpu().numpy() for k, p in model.named_parameters()}
    res = out.detach().double().cpu().numpy(), float(loss), grads
    del model
    torch.cuda.empty_cache()
    return res


def _record(line):
    # measured values of the bounds below, kept next to the other GPU artefacts when the scratch directory exists
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    if os.path.isdir(d):
        with open(os.path.join(d, "northstar_measured.txt"), "a") as f:
            f.write(line + "\n")


def _rel(a, b):
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


def _check_split(pkg, o):
    logits, dice, grads = _ours(pkg, o, "split")
    norm_dev = max(abs(np.linalg.norm(g) / np.linalg.norm(o["grads"][k]) - 1.0) for k, g in grads.items() if np.linalg.norm(o["grads"][k]) > 0)
    _record("split mode vs fp32 oracle: logits rel-L2 %.3e, dice diff %.3e, worst norm deviation %.3e"
            % (_rel(logits, o["logits"]), abs(dice - o["dice"]), norm_dev))
    assert _rel(logits, o["logits"]) < 1e-3                      # north_star logits bound
    assert abs(dice - o["dice"]) < 1e-3 * abs(o["dice"])         # north_star Dice bound
    for k, g in grads.items():
        r = o["grads"][k]
        nr = np.linalg.norm(r)
        assert np.isfinite(g).all(), k
        assert abs(np.linalg.norm(g) - nr) < 3e-2 * nr + 1e-12, (k, np.linalg.norm(g), nr)
        cos = float((g * r).sum() / (np.linalg.norm(g) * nr + 1e-30))
        assert cos > 0.999, (k, cos)


def _check_bf16(pkg, o):
    logits, dice, grads = _ours(pkg, o, "bf16")
    assert abs(dice - o["dice"]) < 1e-3 * abs(o["dice"])
    assert _rel(logits, o["logits"]) < 2e-2                      # measured 4.9e-3 (bf16 operand rounding through 40 layers)
    num = den = 0.0
    for k, g in grads.items():
        r = o["grads"][k]
        assert np.isfinite(g).all(), k
        num += float(((g - r) ** 2).sum())
        den += float((r ** 2).sum())
        if np.linalg.norm(r) > 0:
            assert abs(np.linalg.norm(g) / np.linalg.norm(r) - 1.0) < 5e-2, (k, np.linalg.norm(g), np.linalg.norm(r))
    whole = (num / den) ** 0.5
    worst = max(abs(np.linalg.norm(g) / np.linalg.norm(o["grads"][k]) - 1.0) for k, g in grads.items() if np.linalg.norm(o["grads"][k]) > 0)
    _record("bf16 mode vs fp64 oracle: logits rel-L2 %.3e, dice diff %.3e, whole-gradient rel-L2 %.3e, worst norm deviation %.3e"
            % (_rel(logits, o["logits"]), abs(dice - o["dice"]), whole, worst))
    assert whole < 3e-2              # measured 5.6e-3 (C2) / 6.7e-3 (C3 crop); worst norm deviation measured 3.1e-3 / 5.7e-3


def test_c2_size_split_precision_matches_cpu_oracle(pkg, oracle_c2):
    _check_split(pkg, oracle_c2)


def test_c2_size_bf16_mode_matches_cpu_oracle(pkg, oracle_c2):
    _check_bf16(pkg, oracle_c2)


def test_c3_size_split_precision_matches_cpu_oracle(pkg, oracle_c3):
    _check_split(pkg, oracle_c3)


def test_c3_size_bf16_mode_matches_cpu_oracle(pkg, oracle_c3):
    _check_bf16(pkg, oracle_c3)


def test_c3_shaped_crop_split_precision_matches_cpu_oracle(pkg, oracle_c3crop):
    _check_split(pkg, oracle_c3crop)


def test_c3_shaped_crop_bf16_mode_matches_cpu_oracle(pkg, oracle_c3crop):
    _check_bf16(pkg, oracle_c3crop)
