"""Many-class heads on the host: the oracle against the reference's multi-class fixture (tests/golden/multiclass.npz), the
plans of 9..128-output UNet3D and DynUNet models (parameter spec, the 128-output limit, workspace growth) and the host
layer's marshalling of a 104-output model and of 104-channel pre/post-processing against the stub library."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import UNetConfig, make_state_dict, unet3d_forward, dice_loss
from oracle.prepost_oracle import one_hot_encode, label_map_from_one_hot

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from recipe import golden_inputs, dropout_mask  # noqa: E402
from make_golden_multiclass import (TRAIN_CASES, SOFTMAX_CASE, SHAPE, SUB8, HEAD, N_LABELS, LABEL_MAP_CASES,  # noqa: E402
                                    one_hot_input, label_map_prediction, labels)
from test_dryrun_marshalling import stubbed, fake  # noqa: E402,F401  (stubbed is a fixture)


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "multiclass.npz"))


@pytest.mark.parametrize("name", sorted(TRAIN_CASES))
def test_oracle_matches_multiclass_fixture(name, gold):
    kw = TRAIN_CASES[name]
    cfg = UNetConfig(**kw)
    sd = {k: v.requires_grad_(True) for k, v in make_state_dict(cfg, seed=0, dtype=torch.float64).items()}
    x, t, g3 = golden_inputs(SHAPE, cfg.n_outputs)
    mask = dropout_mask(SHAPE[0], cfg.enc_widths()[0], cfg.dropout, g3)
    logits = unet3d_forward(sd, x.double(), cfg, dropout_mask=mask)
    loss = dice_loss(logits, t)
    loss.backward()
    logits = logits.detach()
    np.testing.assert_allclose(logits[SUB8].numpy(), gold[name + "::logits_sub8"], rtol=0, atol=2e-6)
    assert abs(float(logits.norm()) - float(gold[name + "::logits_norm"])) <= 2e-6 * float(gold[name + "::logits_norm"])
    assert abs(float(loss) - float(gold[name + "::dice"])) <= 2e-6
    keys = list(gold[name + "::grad_keys"])
    assert keys == sorted(sd)
    np.testing.assert_allclose([float(sd[k].grad.norm()) for k in keys], gold[name + "::grad_norms"], rtol=2e-6)
    head = gold[name + "::grad_head"]
    assert head.shape == (cfg.n_outputs, cfg.base_width, 1, 1, 1)
    np.testing.assert_allclose(sd[HEAD].grad.numpy(), head, rtol=0, atol=2e-6 * float(np.abs(head).max()))


def test_oracle_softmax_eval_matches_multiclass_fixture(gold):
    name, kw = SOFTMAX_CASE
    cfg = UNetConfig(**kw)
    x, _, _ = golden_inputs(SHAPE, cfg.n_outputs)
    with torch.no_grad():
        p = unet3d_forward(make_state_dict(cfg, seed=0, dtype=torch.float64), x.double(), cfg)
    np.testing.assert_allclose(p[SUB8].numpy(), gold[name + "::sub8"], rtol=0, atol=2e-6)
    np.testing.assert_allclose(p.sum(dim=1).numpy(), 1.0, atol=1e-12)


def test_prepost_oracle_matches_104_label_fixture(gold):
    y = one_hot_encode(one_hot_input().numpy(), N_LABELS)
    assert tuple(gold["one_hot104_shape"]) == y.shape
    np.testing.assert_array_equal(np.packbits(y.astype(np.uint8)), gold["one_hot104"])
    for name, kw in LABEL_MAP_CASES.items():
        lm = label_map_from_one_hot(label_map_prediction().numpy(), labels(), **kw)
        np.testing.assert_array_equal(lm, gold[name])


# ------------------------------------------------------------------------------------------------ plans
def _unet_plan(pkg, n_outputs, shape=(1, 4, 16, 16, 16), **flags):
    net = pkg.UNet3D(n_features=shape[1], n_outputs=n_outputs, base_width=8)
    desc = net._net_desc(shape[0], *shape[2:])
    for k, v in flags.items():
        setattr(desc, k, v)
    return net, pkg.models._Plan(desc, torch.device("cpu"))


def _dynunet(pkg, out_channels, filters=(8, 16, 24)):
    return pkg.DynUNet(spatial_dims=3, in_channels=4, out_channels=out_channels, kernel_size=[[3, 3, 3]] * len(filters),
                       strides=[[1, 1, 1]] + [[2, 2, 2]] * (len(filters) - 1), upsample_kernel_size=[[2, 2, 2]] * (len(filters) - 1),
                       filters=list(filters))


def _module_spec(net):
    return [(k, tuple(v.shape)) for k, v in net.state_dict().items()]


@pytest.mark.parametrize("n_outputs", [9, 24, 104, 128])
@pytest.mark.parametrize("split", [0, 1])
def test_unet3d_plan_spec_matches_module(pkg, n_outputs, split):
    net, plan = _unet_plan(pkg, n_outputs, split_precision=split)
    assert [(k, tuple(s)) for k, s in plan.param_spec()] == _module_spec(net)
    _, infer = _unet_plan(pkg, n_outputs, split_precision=split, inference_only=1)
    assert infer.param_spec() == plan.param_spec()


@pytest.mark.parametrize("out_channels", [14, 105])
def test_dynunet_plan_spec_matches_module(pkg, out_channels):
    net = _dynunet(pkg, out_channels)
    plan = pkg.models._Plan(net._net_desc(1, 16, 16, 16), torch.device("cpu"))
    assert [(k, tuple(s)) for k, s in plan.param_spec()] == _module_spec(net)
    assert ("output_block.conv.conv.bias", (out_channels,)) in [(k, tuple(s)) for k, s in plan.param_spec()]


def test_129_outputs_are_refused_with_the_limit(pkg):
    with pytest.raises(RuntimeError, match=r"n_outputs=129 unsupported \(1\.\.128\)"):
        _unet_plan(pkg, 129)
    net = _dynunet(pkg, 129)
    with pytest.raises(RuntimeError, match=r"out_channels=129 unsupported \(1\.\.128\)"):
        pkg.models._Plan(net._net_desc(1, 16, 16, 16), torch.device("cpu"))


def test_more_than_8_outputs_need_at_most_64_head_channels(pkg):
    net = pkg.UNet3D(n_features=4, n_outputs=9, base_width=72)
    with pytest.raises(RuntimeError, match="at most 64 channels into the head"):
        pkg.models._Plan(net._net_desc(1, 16, 16, 16), torch.device("cpu"))
    net = pkg.UNet3D(n_features=4, n_outputs=8, base_width=72)                   # the SIMT head takes any width
    pkg.models._Plan(net._net_desc(1, 16, 16, 16), torch.device("cpu"))


@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("flags", [{}, {"deterministic": 1}, {"input_grad": 1}])
def test_104_output_workspace_grows_by_the_head_scratch_alone(pkg, split, flags):
    lib = pkg.lib.load_library()
    _, p3 = _unet_plan(pkg, 3, split_precision=split, **flags)
    _, p104 = _unet_plan(pkg, 104, split_precision=split, **flags)
    scratch = int(lib.b200unet_head_bwd_scratch_bytes(104, 8)) - int(lib.b200unet_head_bwd_scratch_bytes(3, 8))
    growth = p104.ws_bytes - p3.ws_bytes
    assert 0 <= growth <= scratch + 1024, (growth, scratch)
    _, i3 = _unet_plan(pkg, 3, split_precision=split, inference_only=1)
    _, i104 = _unet_plan(pkg, 104, split_precision=split, inference_only=1)
    assert i104.ws_bytes == i3.ws_bytes                                          # no head scratch without a backward


def test_head_scratch_bytes_by_path(pkg):
    lib = pkg.lib.load_library()
    for n_out, c in [(1, 8), (3, 32), (8, 64)]:                                  # SIMT head: one slot per block, 1184 blocks
        assert lib.b200unet_head_bwd_scratch_bytes(n_out, c) == 1184 * n_out * c * 4
    for n_out, c in [(9, 8), (104, 32), (128, 64)]:                              # tensor-core head: dw and dbias slots of 132 CTAs
        assert lib.b200unet_head_bwd_scratch_bytes(n_out, c) == 132 * (n_out * c + n_out) * 4


# ------------------------------------------------------------------------------------------------ host layer (stub library)
def test_104_output_unet3d_training_and_inference_calls(pkg, stubbed):
    model = pkg.UNet3D(n_features=4, n_outputs=104, base_width=8)
    x = fake(torch.randn(1, 4, 16, 16, 16))
    t = fake((torch.rand(1, 104, 16, 16, 16) > 0.5).to(torch.uint8))
    model.train()
    out = model(x)
    assert out.shape == (1, 104, 16, 16, 16) and out.requires_grad
    pkg.DiceLoss(sigmoid=True)(fake(out), t).backward()
    assert all(p.grad is not None and p.grad.shape == p.shape for p in model.parameters())
    assert stubbed.count("b200unet_plan_forward") == 1 and stubbed.count("b200unet_plan_backward") == 1
    assert "b200unet_dice_fwd" in stubbed and "b200unet_dice_bwd" in stubbed
    with torch.no_grad():
        model.eval()
        assert model(x).shape == (1, 104, 16, 16, 16)
    net = _dynunet(pkg, 105)
    net.train()
    net(x).sum().backward()
    assert net.output_block.conv.conv.bias.grad.shape == (105,)


def test_104_channel_prepost_calls(pkg, stubbed):
    lab = fake(torch.randint(0, 105, (1, 1, 6, 6, 6)).float())
    assert pkg.prepost.compile_one_hot_encoding(lab, n_labels=104).shape == (104, 6, 6, 6)
    p = fake(torch.rand(104, 6, 6, 6))
    assert pkg.prepost.convert_one_hot_to_label_map(p, labels(), activation="softmax").shape == (6, 6, 6)
    assert pkg.prepost.convert_one_hot_to_label_map_using_hierarchy(p, labels()).shape == (6, 6, 6)
    assert stubbed.count("b200unet_one_hot") == 1 and stubbed.count("b200unet_label_map") == 2
