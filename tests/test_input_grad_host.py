"""Input gradient (d(loss)/d(x)) without a GPU: the oracle restatement against the reference's own input gradient
(tests/golden/input_grad.npz, tests/golden/make_golden_input_grad.py), the plan's workspace and parameter spec with and
without ``input_grad``, and the host layer's autograd plumbing against the marshalling stub of test_dryrun_marshalling."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import UNetConfig, make_state_dict, unet3d_forward, dice_loss

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from recipe import CASES, golden_inputs, dropout_mask  # noqa: E402
from make_golden_input_grad import INPUT_GRAD_CASES, SUB  # noqa: E402
from test_dryrun_marshalling import stubbed, fake, _FakeCuda  # noqa: E402,F401  (stubbed is a fixture)

FAST = ["c1_bw8_32", "bw16_n2_32", "bw8_convT_32", "c5like_1ch_5lev_32", "bw8_nonpow2_24x32x40", "identity_bw8_n8_32"]


def oracle_input_grad(kw, shape, dtype=torch.float64):
    """autograd input gradient of the oracle restatement, train mode with the recipe's dropout mask"""
    cfg = UNetConfig(**kw)
    sd = make_state_dict(cfg, seed=0, dtype=dtype)
    x, t, g3 = golden_inputs(shape, cfg.n_outputs)
    x = x.to(dtype).requires_grad_(True)
    mask = dropout_mask(shape[0], cfg.enc_widths()[0], cfg.dropout, g3)
    dice_loss(unet3d_forward(sd, x, cfg, dropout_mask=mask), t).backward()
    return x.grad


@pytest.mark.parametrize("name", FAST)
def test_oracle_input_gradient_matches_reference_fixture(name, golden_dir):
    gold = np.load(os.path.join(golden_dir, "input_grad.npz"))
    dx = oracle_input_grad(*INPUT_GRAD_CASES[name])
    scale = float(np.abs(gold[name + "::sub4"]).max())
    np.testing.assert_allclose(dx[SUB].numpy(), gold[name + "::sub4"], rtol=0, atol=2e-6 * scale)
    assert abs(float(dx.norm()) - float(gold[name + "::norm"])) <= 2e-6 * float(gold[name + "::norm"])
    np.testing.assert_allclose(dx.flatten(2).norm(dim=2).numpy(), gold[name + "::nc_norms"], rtol=2e-6)


def test_fixture_covers_every_recipe_case_and_the_identity_branch(golden_dir):
    gold = np.load(os.path.join(golden_dir, "input_grad.npz"))
    assert set(CASES) < set(INPUT_GRAD_CASES)
    for name, (kw, shape) in INPUT_GRAD_CASES.items():
        assert gold[name + "::nc_norms"].shape == (shape[0], shape[1])
        assert float(gold[name + "::norm"]) > 0
    kw = INPUT_GRAD_CASES["identity_bw8_n8_32"][0]
    assert kw["n_features"] == kw["base_width"]


# ------------------------------------------------------------------------------------------------ plan: ABI and workspace
def _unet(pkg, kw, shape, **flags):
    net = pkg.UNet3D(**kw)
    desc = net._net_desc(shape[0], *shape[2:])
    for k, v in flags.items():
        setattr(desc, k, v)
    return pkg.models._Plan(desc, torch.device("cpu"))


BRATS_DYNUNET = dict(spatial_dims=3, in_channels=4, out_channels=3, kernel_size=[[3, 3, 3]] * 6, strides=[[1, 1, 1]] + [[2, 2, 2]] * 5,
                     upsample_kernel_size=[[2, 2, 2]] * 5, filters=[64, 96, 128, 192, 256, 384])


def _ceil(v, m):
    return (v + m - 1) // m * m


@pytest.mark.parametrize("name", list(INPUT_GRAD_CASES) + ["nf12_bw16", "nf16_bw16"])
@pytest.mark.parametrize("split", [0, 1])
def test_flagged_unet3d_plan_same_spec_and_only_the_new_buffers(pkg, name, split):
    kw, shape = INPUT_GRAD_CASES.get(name, (None, None))
    if name == "nf12_bw16":
        kw, shape = dict(n_features=12, n_outputs=2, base_width=16), (2, 12, 16, 16, 16)
    elif name == "nf16_bw16":
        kw, shape = dict(n_features=16, n_outputs=2, base_width=16), (1, 16, 16, 16, 16)
    plain = _unet(pkg, kw, shape, split_precision=split)
    flagged = _unet(pkg, kw, shape, split_precision=split, input_grad=1)
    assert flagged.param_spec() == plain.param_spec()
    growth = flagged.ws_bytes - plain.ws_bytes
    n, cin = shape[0], shape[1]
    cp = _ceil(cin, 8)
    copies = 2 if split else 1
    if cin == kw["base_width"]:
        new = []                                       # identity branch: the dgrad pack of conv1 exists already, no buffer
    else:                                              # 1x1x1 `sample` data-gradient pack [1][Cip][Cop] + its 8/16-channel output
        new = [cp * kw["base_width"] * 2] * copies + [n * int(np.prod(shape[2:])) * cp * 2] * copies
    assert growth >= 0
    assert abs(growth - sum(new)) <= 1024 * (len(new) + 1), (growth, new)
    if not new:
        assert growth == 0


@pytest.mark.parametrize("kw,shape", [
    (dict(spatial_dims=3, in_channels=4, out_channels=3, kernel_size=[[3, 3, 3]] * 3, strides=[[1, 1, 1]] + [[2, 2, 2]] * 2,
          upsample_kernel_size=[[2, 2, 2]] * 2, filters=[8, 16, 24]), (1, 4, 16, 16, 16)),
    (dict(spatial_dims=3, in_channels=12, out_channels=2, kernel_size=[[3, 3, 3]] * 3, strides=[[1, 1, 1]] + [[2, 2, 2]] * 2,
          upsample_kernel_size=[[2, 2, 2]] * 2, filters=[16, 24, 32]), (2, 12, 16, 16, 16)),
    (BRATS_DYNUNET, (2, 4, 128, 128, 128)),
])
def test_flagged_dynunet_plan_same_spec_and_only_the_new_buffers(pkg, kw, shape):
    net = pkg.DynUNet(**kw)
    desc = net._net_desc(shape[0], *shape[2:])
    plain = pkg.models._Plan(desc, torch.device("cpu"))
    desc.input_grad = 1
    flagged = pkg.models._Plan(desc, torch.device("cpu"))
    assert flagged.param_spec() == plain.param_spec()
    cp = _ceil(shape[1], 8)
    new = [27 * cp * kw["filters"][0] * 2, shape[0] * int(np.prod(shape[2:])) * cp * 2]   # conv1 data-gradient pack, dX buffer
    growth = flagged.ws_bytes - plain.ws_bytes
    assert growth >= 0 and abs(growth - sum(new)) <= 1024 * (len(new) + 1), (growth, new)


def test_inference_only_plan_with_input_grad_is_refused(pkg):
    kw, shape = CASES["c1_bw8_32"]
    with pytest.raises(RuntimeError, match="input_grad=1 on an inference_only plan"):
        _unet(pkg, kw, shape, inference_only=1, input_grad=1)
    net = pkg.DynUNet(**BRATS_DYNUNET)
    desc = net._net_desc(1, 64, 64, 64)
    desc.inference_only, desc.input_grad = 1, 1
    with pytest.raises(RuntimeError, match="inference_only"):
        pkg.models._Plan(desc, torch.device("cpu"))


def test_input_grad_entry_point_needs_a_flagged_plan(pkg):
    kw, shape = CASES["c1_bw8_32"]
    plan = _unet(pkg, kw, shape)
    lib = pkg.lib.load_library()
    assert lib.b200unet_plan_input_grad(plan.handle, 8, 8, None) != 0           # rejected before any device access
    assert "without input_grad" in lib.b200unet_last_error().decode()


# ------------------------------------------------------------------------------------------------ host layer (stub library)
def _x(shape=(1, 4, 16, 16, 16)):
    return fake(torch.randn(shape)).requires_grad_(True)


def test_unet3d_input_gradient_call_follows_the_backward(pkg, stubbed):
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=8)
    model.train()
    x = _x()
    model(x).sum().backward()
    calls = [c for c in stubbed if c.startswith("b200unet_plan_")]
    assert calls == ["b200unet_plan_forward", "b200unet_plan_backward", "b200unet_plan_input_grad"]
    assert x.grad is not None and x.grad.shape == x.shape and x.grad.dtype == x.dtype
    assert all(p.grad is not None for p in model.parameters())
    assert [k[-2:] for k in model._plans] == [(True, False)]                   # (input_grad, inference_only)
    # without an input that needs a gradient: the unflagged plan, no input-gradient call
    del stubbed[:]
    model(fake(torch.randn(1, 4, 16, 16, 16))).sum().backward()
    assert "b200unet_plan_input_grad" not in stubbed and stubbed.count("b200unet_plan_backward") == 1
    assert sorted(k[-2:] for k in model._plans) == [(False, False), (True, False)]
    # no_grad: the forward-only plan, whatever the input
    with torch.no_grad():
        model(x)
    assert (False, True) in [k[-2:] for k in model._plans]


def test_frozen_parameters_still_give_the_input_gradient(pkg, stubbed):
    """saliency maps of a trained, frozen network: only the input asks for a gradient"""
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=8)
    model.eval()
    for p in model.parameters():
        p.requires_grad_(False)
    x = _x()
    model(x).sum().backward()
    assert x.grad is not None and x.grad.shape == x.shape
    assert stubbed.count("b200unet_plan_input_grad") == 1


def test_input_gradient_reaches_non_float_and_non_contiguous_inputs(pkg, stubbed):
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=8)
    x = fake(torch.randn(1, 16, 16, 16, 4, dtype=torch.float64)).requires_grad_(True)
    model(x.permute(0, 4, 1, 2, 3)).sum().backward()
    assert x.grad is not None and x.grad.shape == x.shape and x.grad.dtype == torch.float64


def test_autoimplant_input_gets_a_gradient(pkg, stubbed):
    model = pkg.AutoImplantUNet(n_features=3, n_outputs=3, base_width=8)
    x = _x((1, 3, 16, 16, 16))
    model(x).sum().backward()
    assert x.grad is not None and x.grad.shape == x.shape
    assert stubbed.count("b200unet_plan_input_grad") == 1


class _MetaLike(_FakeCuda):
    """a torch.Tensor subclass that carries metadata, as MONAI's MetaTensor does"""
    meta = {"affine": None}


def test_metatensor_like_input_receives_grad(pkg, stubbed):
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=8)
    x = torch.randn(1, 4, 16, 16, 16).as_subclass(_MetaLike).requires_grad_(True)
    model(x).sum().backward()
    assert x.grad is not None and x.grad.shape == x.shape
    assert stubbed.count("b200unet_plan_input_grad") == 1


def test_dynunet_input_gradient_calls(pkg, stubbed):
    model = pkg.DynUNet(spatial_dims=3, in_channels=4, out_channels=3, kernel_size=[[3, 3, 3]] * 3,
                        strides=[[1, 1, 1], [2, 2, 2], [2, 2, 2]], upsample_kernel_size=[[2, 2, 2]] * 2, filters=[8, 16, 24])
    model.train()
    x = _x()
    model(x).sum().backward()
    assert [c for c in stubbed if c.startswith("b200unet_plan_")][-2:] == ["b200unet_plan_backward", "b200unet_plan_input_grad"]
    assert x.grad.shape == x.shape


def test_flat_gradients_with_an_input_gradient_calls(pkg, stubbed):
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=8)
    model.train()
    model.use_flat_gradients(True)
    x = _x()
    model(x).sum().backward()
    assert stubbed.count("b200unet_plan_backward") == 1 and stubbed.count("b200unet_plan_input_grad") == 1
    assert x.grad is not None


def test_double_backward_through_the_input_gradient_raises(pkg, stubbed):
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=8)
    x = _x()
    with pytest.raises(RuntimeError, match="double backward"):
        torch.autograd.grad(model(x).sum(), x, create_graph=True)


def test_one_outstanding_forward_guard_applies_to_flagged_plans(pkg, stubbed):
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=8)
    x = _x()
    o1 = model(x)
    o2 = model(x)
    o2.sum().backward()
    with pytest.raises(RuntimeError, match="overwritten the saved activations"):
        o1.sum().backward()
