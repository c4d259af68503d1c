"""Whole-path parity on the GPU: the GPU UNet3D + fused Dice, called through the reference-facing module API
(which goes through the C-ABI plan), against (a) the committed golden fixtures produced by the unmodified
reference, (b) the CPU oracle, and (c) size-independent properties at BASELINE.json's full 128^3 size.

Tolerances (north_star): logits and Dice within 1e-3 relative of the fp32 reference -- claimed in `split`
precision (hi/lo bf16 operands, 3 MMAs); in single-pass `bf16` the Dice bound holds and logits carry the bf16
operand noise (~1e-2, SURVEY.md section 0), gradients ~1e-1 like torch's own bf16 autocast."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import UNetConfig, make_state_dict, unet3d_forward, dice_loss, sliding_window_inference

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from recipe import CASES, golden_inputs, dropout_mask  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SUB = (slice(None), slice(None), slice(None, None, 4), slice(None, None, 4), slice(None, None, 4))


def _run(pkg, name, precision):
    kw, shape = CASES[name]
    cfg = UNetConfig(**kw)
    model = pkg.UNet3D(precision=precision, **kw).to(DEV)
    model.load_state_dict(make_state_dict(cfg, seed=0), strict=True)
    x, t, g3 = golden_inputs(shape, cfg.n_outputs)
    mask = dropout_mask(shape[0], cfg.enc_widths()[0], cfg.dropout, g3)
    model.train()
    model.set_dropout_scale(mask)
    crit = pkg.DiceLoss(sigmoid=True)
    out = model(x.to(DEV))
    loss = crit(out, t.to(DEV))
    loss.backward()
    model.eval()
    with torch.no_grad():
        out_eval = model(x.to(DEV))
    torch.cuda.synchronize()
    return model, out.detach().cpu(), float(loss), out_eval.cpu()


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


@pytest.mark.parametrize("name", ["c1_bw8_32", "c1_bw8_64", "bw16_n2_32", "c5like_1ch_5lev_32", "bw8_nonpow2_24x32x40",
                                  "bw8_convT_32"])
def test_split_precision_matches_reference_goldens(pkg, golden_dir, name):
    gold = np.load(os.path.join(golden_dir, name + ".npz"))
    model, out, loss, out_eval = _run(pkg, name, "split")
    assert _rel(out[SUB].numpy(), gold["logits_sub4"]) < 1e-3          # north_star logits bound (measured ~2e-5)
    assert _rel(out_eval[SUB].numpy(), gold["logits_eval_sub4"]) < 1e-3
    assert abs(float(out.double().norm()) - float(gold["logits_norm"])) < 1e-3 * float(gold["logits_norm"])
    assert abs(loss - float(gold["dice"])) < 1e-3 * float(gold["dice"])  # north_star Dice bound (measured ~1e-8)
    norms = dict(zip([str(k) for k in gold["grad_keys"]], gold["grad_norms"]))
    for k, p in model.named_parameters():
        g = p.grad.double().cpu().numpy()
        assert np.isfinite(g).all(), k
        assert abs(np.linalg.norm(g) - norms[k]) < 3e-2 * norms[k] + 1e-12, k        # chaotic amplification ~1e-3..1e-2
        gk = "grad::" + k
        if gk in gold and norms[k] > 0:
            cos = float((g * gold[gk]).sum() / (np.linalg.norm(g) * np.linalg.norm(gold[gk]) + 1e-30))
            assert cos > 0.999, (k, cos)


@pytest.mark.parametrize("name", ["c1_bw8_32", "bw16_n2_32"])
def test_bf16_mode_dice_bound_and_logit_noise(pkg, golden_dir, name):
    gold = np.load(os.path.join(golden_dir, name + ".npz"))
    model, out, loss, out_eval = _run(pkg, name, "bf16")
    assert abs(loss - float(gold["dice"])) < 1e-3 * float(gold["dice"])
    assert _rel(out[SUB].numpy(), gold["logits_sub4"]) < 4e-2
    norms = dict(zip([str(k) for k in gold["grad_keys"]], gold["grad_norms"]))
    for k, p in model.named_parameters():
        g = p.grad.double().cpu().numpy()
        assert np.isfinite(g).all(), k
        gk = "grad::" + k
        if gk in gold and norms[k] > 0:
            cos = float((g * gold[gk]).sum() / (np.linalg.norm(g) * np.linalg.norm(gold[gk]) + 1e-30))
            assert cos > 0.9, (k, cos)


def test_oracle_parity_with_encoder_variants(pkg):
    """block counts that exercise dropout landing mid-level (encoder_blocks[0] = 2) and deeper decoders."""
    kw = dict(n_features=2, n_outputs=2, base_width=8, encoder_blocks=[2, 1, 2], decoder_blocks=[1, 2, 2])
    cfg = UNetConfig(**kw)
    sd = make_state_dict(cfg, seed=4)
    shape = (2, 2, 16, 24, 16)
    x, t, g3 = golden_inputs(shape, cfg.n_outputs, seed=11)
    mask = dropout_mask(2, 8, 0.2, g3)
    sd64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    ref = unet3d_forward(sd64, x.double(), cfg, dropout_mask=mask)
    lref = dice_loss(ref, t)
    lref.backward()
    model = pkg.UNet3D(precision="split", **kw).to(DEV)
    model.load_state_dict(sd, strict=True)
    model.train()
    model.set_dropout_scale(mask)
    out = model(x.to(DEV))
    loss = pkg.DiceLoss(sigmoid=True)(out, t.to(DEV))
    loss.backward()
    assert _rel(out.detach().cpu().numpy(), ref.detach().numpy()) < 1e-3
    assert abs(float(loss) - float(lref)) < 1e-5
    for k, p in model.named_parameters():
        r = _rel(p.grad.cpu().numpy(), sd64[k].grad.numpy())
        assert r < 5e-2, (k, r)


def test_no_input_gradient_and_shape_errors(pkg):
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=8).to(DEV)
    with pytest.raises(ValueError):
        model(torch.zeros(1, 3, 16, 16, 16, device=DEV))
    with pytest.raises(RuntimeError, match="must be even"):
        model(torch.zeros(1, 4, 20, 16, 16, device=DEV))              # 20 -> 10 -> 5 (odd) before the last level


def test_sliding_window_inference_matches_oracle(pkg):
    """config-5 style tiled inference (1-channel, 5 levels) through the on-device inferer vs the oracle inferer
    driving the oracle model on the CPU."""
    kw = dict(n_features=1, n_outputs=1, base_width=8, encoder_blocks=[1, 1, 1, 1, 1])
    cfg = UNetConfig(**kw)
    sd = make_state_dict(cfg, seed=2)
    x = torch.randn(1, 1, 48, 48, 48, generator=torch.Generator().manual_seed(3))
    model = pkg.UNet3D(precision="split", **kw).to(DEV)
    model.load_state_dict(sd, strict=True)
    model.eval()
    inf = pkg.predict.SlidingWindowInferer(roi_size=(32, 32, 32), sw_batch_size=2, overlap=0.25, mode="gaussian")
    with torch.no_grad():
        got = inf(x.to(DEV), model).cpu()
        sd64 = {k: v.double() for k, v in sd.items()}
        ref = sliding_window_inference(x.double(), (32, 32, 32), lambda p: unet3d_forward(sd64, p, cfg), overlap=0.25, mode="gaussian")
    assert _rel(got.numpy(), ref.numpy()) < 1e-3


# ------------------------------------------------------------------------------------------------ full size (C2) properties
@pytest.fixture(scope="module")
def c2(pkg):
    torch.manual_seed(0)
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=32, precision="bf16").to(DEV)
    x = torch.randn(2, 4, 128, 128, 128, device=DEV)
    t = (torch.rand(2, 3, 128, 128, 128, device=DEV) > 0.7).to(torch.uint8)
    return model, x, t


def test_c2_full_size_dice_matches_oracle_on_same_logits(pkg, c2):
    model, x, t = c2
    model.eval()
    with torch.no_grad():
        out = model(x)
    loss = pkg.DiceLoss(sigmoid=True)(out, t)
    ref = dice_loss(out.double().cpu(), t.cpu())                      # oracle Dice over 2x3x128^3 voxels
    assert torch.isfinite(out).all()
    assert abs(float(loss) - float(ref)) < 1e-6


def test_c2_full_size_samples_are_independent(pkg, c2):
    """GroupNorm and Dice are per-sample: swapping the batch order must swap the outputs (the property that makes
    the path shard over GPUs without a forward exchange).  The two runs reduce the GroupNorm statistics in a
    different order (persistent CTAs, fp32 partial sums), so in bf16 storage individual roundings flip and are
    amplified like any other bf16 noise (~1e-2); in split precision the same comparison is tight."""
    model, x, t = c2
    model.eval()
    with torch.no_grad():
        a = model(x)
        b = model(x.flip(0).contiguous())
    assert float((a - b.flip(0)).norm() / a.norm()) < 2e-2
    model_s = pkg.UNet3D(n_features=4, n_outputs=3, base_width=32, precision="split").to(DEV)
    model_s.load_state_dict(model.state_dict())
    model_s.eval()
    with torch.no_grad():
        a = model_s(x)
        b = model_s(x.flip(0).contiguous())
    assert float((a - b.flip(0)).norm() / a.norm()) < 1e-4


def test_c2_full_size_backward_is_linear_in_dlogits(pkg, c2):
    model, x, t = c2
    model.train()
    model.set_dropout_scale(torch.ones(2, 32))
    g = torch.randn(2, 3, 128, 128, 128, device=DEV) * 1e-6
    model.zero_grad(set_to_none=True)
    model(x).backward(g)
    g1 = [p.grad.clone() for p in model.parameters()]
    model.zero_grad(set_to_none=True)
    model(x).backward(2.0 * g)                                        # power-of-two scale: exact in bf16/fp32
    g2 = [p.grad for p in model.parameters()]
    num = sum(float((2.0 * a - b).double().pow(2).sum()) for a, b in zip(g1, g2)) ** 0.5
    den = sum(float(b.double().pow(2).sum()) for b in g2) ** 0.5
    assert num / den < 2e-3                       # whole gradient vector
    for a, b in zip(g1, g2):
        assert torch.isfinite(b).all()
        # per tensor: sums with heavy cancellation (GroupNorm beta/gamma of the first layers) see the
        # run-to-run order of the fp32 partial-sum atomics
        assert float((2.0 * a - b).norm() / (b.norm() + 1e-30)) < 5e-2
