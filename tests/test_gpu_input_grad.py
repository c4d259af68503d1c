"""Input gradient on the GPU (``b200unet_plan_input_grad`` through the module API): split precision against the gradient the
UNMODIFIED reference produces for its input (tests/golden/input_grad.npz), bf16 against torch's own bf16 autocast, DynUNet
against its (unpinned) oracle, and the properties that do not need a reference: flagged plans leave the parameter gradients
bit for bit unchanged, determinism, linearity in dlogits, batch-order equivariance, the flat-gradient setup, AutoImplantUNet."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import UNetConfig, make_state_dict, unet3d_forward, dice_loss
from oracle.dynunet_oracle import make_dynunet_state_dict, dynunet_forward

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from recipe import golden_inputs, dropout_mask  # noqa: E402
from make_golden_input_grad import INPUT_GRAD_CASES, SUB  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


def _cos(a, b):
    a, b = np.asarray(a, dtype=np.float64).ravel(), np.asarray(b, dtype=np.float64).ravel()
    return float((a * b).sum() / (np.linalg.norm(a) * np.linalg.norm(b) + 1e-300))


def _golden_run(pkg, kw, shape, precision="split", deterministic=None):
    cfg = UNetConfig(**kw)
    model = pkg.UNet3D(precision=precision, deterministic=deterministic, **kw).to(DEV)
    model.load_state_dict(make_state_dict(cfg, seed=0), strict=True)
    x, t, g3 = golden_inputs(shape, cfg.n_outputs)
    model.train()
    model.set_dropout_scale(dropout_mask(shape[0], cfg.enc_widths()[0], cfg.dropout, g3))
    xd = x.to(DEV).requires_grad_(True)
    pkg.DiceLoss(sigmoid=True)(model(xd), t.to(DEV)).backward()
    torch.cuda.synchronize()
    return model, xd.grad.detach().cpu()


@pytest.mark.parametrize("name", list(INPUT_GRAD_CASES))
def test_split_precision_input_gradient_matches_reference_fixture(pkg, golden_dir, name):
    """the bounds test_gpu_model.py applies to the split-mode parameter gradients: norm within 3 %, cosine > 0.999"""
    gold = np.load(os.path.join(golden_dir, "input_grad.npz"))
    _, dx = _golden_run(pkg, *INPUT_GRAD_CASES[name])
    assert torch.isfinite(dx).all()
    norm, gnorm = float(dx.double().norm()), float(gold[name + "::norm"])
    print("%s: |dx| %.6e vs reference %.6e (ratio %.5f), cosine of the stride-4 sample %.6f"
          % (name, norm, gnorm, norm / gnorm, _cos(dx[SUB].numpy(), gold[name + "::sub4"])))
    assert abs(norm - gnorm) < 3e-2 * gnorm
    np.testing.assert_allclose(dx.double().flatten(2).norm(dim=2).numpy(), gold[name + "::nc_norms"], rtol=3e-2)
    assert _cos(dx[SUB].numpy(), gold[name + "::sub4"]) > 0.999


@pytest.mark.parametrize("kw,shape", [(dict(n_features=12, n_outputs=2, base_width=16), (2, 12, 32, 32, 32)),
                                      (dict(n_features=16, n_outputs=2, base_width=16), (1, 16, 32, 32, 32)),
                                      (dict(n_features=2, n_outputs=2, base_width=8, encoder_blocks=[2, 1, 2]), (2, 2, 16, 24, 16))])
def test_split_precision_input_gradient_matches_oracle_autograd(pkg, kw, shape):
    """16 padded input channels (sample branch and identity branch), and dropout landing on block (0, 1)'s input"""
    cfg = UNetConfig(**kw)
    sd = make_state_dict(cfg, seed=4)
    x, t, g3 = golden_inputs(shape, cfg.n_outputs, seed=11)
    mask = dropout_mask(shape[0], cfg.enc_widths()[0], cfg.dropout, g3)
    x64 = x.double().requires_grad_(True)
    dice_loss(unet3d_forward({k: v.double() for k, v in sd.items()}, x64, cfg, dropout_mask=mask), t).backward()
    model = pkg.UNet3D(precision="split", **kw).to(DEV)
    model.load_state_dict(sd, strict=True)
    model.train()
    model.set_dropout_scale(mask)
    xd = x.to(DEV).requires_grad_(True)
    pkg.DiceLoss(sigmoid=True)(model(xd), t.to(DEV)).backward()
    ref = x64.grad
    assert abs(float(xd.grad.double().norm()) / float(ref.norm()) - 1.0) < 3e-2
    assert _cos(xd.grad.cpu().numpy(), ref.numpy()) > 0.999


def test_bf16_input_gradient_error_is_torch_autocast_class(pkg):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    kw = dict(n_features=4, n_outputs=3, base_width=16)
    cfg = UNetConfig(**kw)
    sd = make_state_dict(cfg, seed=0)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, 4, 64, 64, 64, generator=g)
    t = (torch.rand(1, 3, 64, 64, 64, generator=g) > 0.7).to(torch.uint8)

    def oracle_dx(dtype, autocast):
        sdr = {k: v.to(DEV, dtype) for k, v in sd.items()}
        xr = x.to(DEV, dtype).requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            out = unet3d_forward(sdr, xr, cfg)
        dice_loss(out.float() if autocast else out, t.to(DEV)).backward()
        return xr.grad.double()
    ref, ac = oracle_dx(torch.float64, False), oracle_dx(torch.float32, True)
    model = pkg.UNet3D(precision="bf16", **kw).to(DEV)
    model.load_state_dict(sd, strict=True)
    model.train()
    model.set_dropout_scale(torch.ones(1, 16))
    xd = x.to(DEV).requires_grad_(True)
    pkg.DiceLoss(sigmoid=True)(model(xd), t.to(DEV)).backward()
    ours, theirs = _rel(xd.grad, ref), _rel(ac, ref)
    print("bf16 input gradient rel-L2: ours %.4e, torch bf16 autocast %.4e (ratio %.3f)" % (ours, theirs, ours / theirs))
    assert ours <= 1.25 * theirs


@pytest.mark.parametrize("precision", ["bf16", "split"])
def test_flagged_plan_keeps_parameter_gradients_bit_identical(pkg, precision):
    kw = dict(n_features=4, n_outputs=3, base_width=16)
    sd = make_state_dict(UNetConfig(**kw), seed=9)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 4, 32, 32, 32, generator=g).to(DEV)
    t = (torch.rand(2, 3, 32, 32, 32, generator=g) > 0.7).to(torch.uint8).to(DEV)
    model = pkg.UNet3D(precision=precision, deterministic=True, **kw).to(DEV)
    model.load_state_dict(sd)
    model.train()
    model.set_dropout_scale(torch.ones(2, 16))
    runs, dxs = [], []
    for needs_dx in (False, True, True):
        model.zero_grad(set_to_none=True)
        xi = x.clone().requires_grad_(needs_dx)
        pkg.DiceLoss(sigmoid=True)(model(xi), t).backward()
        runs.append([p.grad.clone() for p in model.ordered_parameters()])
        if needs_dx:
            dxs.append(xi.grad.clone())
    assert sorted(k[-2:] for k in model._plans) == [(False, False), (True, False)]
    for run in runs[1:]:
        for k, a, b in zip(model._keys, runs[0], run):
            assert torch.equal(a, b), k
    assert torch.equal(dxs[0], dxs[1]), "a deterministic plan must repeat its input gradient bit for bit"


def test_input_gradient_is_linear_in_dlogits_and_batch_order_equivariant(pkg):
    torch.manual_seed(0)
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=16, precision="split", deterministic=True).to(DEV)
    model.train()
    model.set_dropout_scale(torch.ones(2, 16))
    x = torch.randn(2, 4, 32, 32, 32, device=DEV)
    gl = torch.randn(2, 3, 32, 32, 32, device=DEV) * 1e-3

    def dx_of(xv, dl):
        xi = xv.clone().requires_grad_(True)
        model(xi).backward(dl)
        return xi.grad
    d1, d2 = dx_of(x, gl), dx_of(x, 2.0 * gl)                    # power-of-two scale: exact in bf16 / fp32
    assert _rel(d2, 2.0 * d1) < 1e-4
    d3 = dx_of(x, gl + 0.5 * gl.flip(0))
    d4 = dx_of(x, 0.5 * gl.flip(0))
    assert _rel(d3 - d4, d1) < 1e-3                              # additivity, up to the rounding of the stored gradients
    df = dx_of(x.flip(0).contiguous(), gl.flip(0).contiguous())
    assert _rel(df.flip(0), d1) < 1e-3


@pytest.mark.parametrize("cin,cout,filters,shape", [(4, 3, [8, 16, 24, 32], (1, 4, 32, 32, 32)), (1, 2, [16, 24, 48], (2, 1, 16, 32, 24)),
                                                    (12, 2, [32, 48, 64], (1, 12, 16, 16, 32))])
def test_dynunet_split_precision_input_gradient_matches_unpinned_oracle(pkg, cin, cout, filters, shape):
    L = len(filters)
    kw = dict(spatial_dims=3, in_channels=cin, out_channels=cout, kernel_size=[[3, 3, 3]] * L, strides=[[1, 1, 1]] + [[2, 2, 2]] * (L - 1),
              upsample_kernel_size=[[2, 2, 2]] * (L - 1), filters=filters)
    sd = make_dynunet_state_dict(cin, cout, filters, seed=1)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(shape, generator=g)
    t = (torch.rand((shape[0], cout) + shape[2:], generator=g) > 0.7).to(torch.uint8)
    x64 = x.double().requires_grad_(True)
    dice_loss(dynunet_forward({k: v.double() for k, v in sd.items()}, x64, L), t).backward()
    model = pkg.DynUNet(precision="split", **kw).to(DEV)
    model.load_state_dict(sd, strict=True)
    model.train()
    xd = x.to(DEV).requires_grad_(True)
    pkg.DiceLoss(sigmoid=True)(model(xd), t.to(DEV)).backward()
    assert abs(float(xd.grad.double().norm()) / float(x64.grad.norm()) - 1.0) < 3e-2
    assert _cos(xd.grad.cpu().numpy(), x64.grad.numpy()) > 0.999


def test_flat_gradients_give_the_same_input_gradient(pkg):
    kw = dict(n_features=2, n_outputs=2, base_width=8)
    sd = make_state_dict(UNetConfig(**kw), seed=3)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 2, 32, 32, 32, generator=g).to(DEV)
    t = (torch.rand(2, 2, 32, 32, 32, generator=g) > 0.6).to(torch.uint8).to(DEV)
    out = {}
    for flat in (False, True):
        model = pkg.UNet3D(precision="bf16", deterministic=True, dropout=0.0, **kw).to(DEV)
        model.load_state_dict(sd)
        model.train()
        if flat:
            model.use_flat_gradients(True)
        xi = x.clone().requires_grad_(True)
        pkg.DiceLoss(sigmoid=True)(model(xi), t).backward()
        out[flat] = (xi.grad.clone(), [p.grad.clone() for p in model.ordered_parameters()])
    assert torch.equal(out[False][0], out[True][0])
    for a, b in zip(out[False][1], out[True][1]):
        assert torch.equal(a, b)


def test_autoimplant_input_gradient_is_unet_gradient_minus_grad_out(pkg):
    kw = dict(n_features=3, n_outputs=3, base_width=8)
    sd = make_state_dict(UNetConfig(**kw), seed=6)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(1, 3, 32, 32, 32, generator=g).to(DEV)
    grad_out = (torch.randn(1, 3, 32, 32, 32, generator=g) * 1e-3).to(DEV)
    dxs = {}
    for cls in (pkg.UNet3D, pkg.AutoImplantUNet):
        model = cls(precision="split", deterministic=True, **kw).to(DEV)
        model.load_state_dict(sd)
        model.train()
        model.set_dropout_scale(torch.ones(1, 8))
        xi = x.clone().requires_grad_(True)
        model(xi).backward(grad_out)
        dxs[cls] = xi.grad
    assert torch.equal(dxs[pkg.AutoImplantUNet], dxs[pkg.UNet3D] - grad_out)
