"""MONAI UNet on the host: the module's state-dict spec equals the oracle's and the library plan's, MONAI's ValueErrors, every
unimplemented option raises NotImplementedError naming it, and the tutorial-size workspaces."""
import pytest
import torch

from oracle.unet_oracle import MonaiUNetConfig, unet_state_dict_spec


def _plan(pkg, m, n, d, h, w, **flags):
    desc = m._net_desc(n, d, h, w)
    for k, v in flags.items():
        setattr(desc, k, v)
    return pkg.models._Plan(desc, torch.device("cpu"))


@pytest.mark.parametrize("r", [0, 1, 2])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("act,affine", [("prelu", False), ("relu", True), ("leakyrelu", False)])
def test_spec_module_oracle_plan_agree(pkg, r, bias, act, affine):
    m = pkg.UNet(in_channels=4, out_channels=3, channels=(16, 32, 64, 64), strides=(2, 2, 2), num_res_units=r, bias=bias, act=act,
                 norm=("instance", {"affine": affine}))
    spec = unet_state_dict_spec(MonaiUNetConfig(4, 3, (16, 32, 64, 64), r, act, norm_affine=affine, bias=bias))
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == spec
    assert m._param_spec_cpu() == spec
    for flags in ({}, {"input_grad": 1}, {"inference_only": 1}, {"split_precision": 1}, {"deterministic": 1}):
        assert _plan(pkg, m, 1, 32, 32, 32, **flags).param_spec() == spec
    sd = {k: torch.randn_like(v) for k, v in m.state_dict().items()}
    m.load_state_dict(sd, strict=True)


def test_monai_key_examples_and_init(pkg):
    m = pkg.UNet(in_channels=1, out_channels=2, channels=(16, 32, 64), strides=(2, 2), num_res_units=2)
    keys = list(m.state_dict())
    for k in ("model.0.conv.unit0.conv.weight", "model.0.conv.unit0.adn.A.weight", "model.0.residual.bias",
              "model.1.submodule.0.conv.unit1.conv.bias", "model.1.submodule.1.submodule.residual.weight",
              "model.2.0.conv.weight", "model.2.1.conv.unit0.conv.bias"):
        assert k in keys, k
    assert "model.2.1.conv.unit0.adn.A.weight" not in keys     # the top unit is conv-only
    assert float(m.state_dict()["model.0.conv.unit0.adn.A.weight"]) == 0.25
    assert float(pkg.UNet(channels=(8, 16), strides=(2,), act=("prelu", {"init": 0.1})).state_dict()["model.0.adn.A.weight"]) == \
        pytest.approx(0.1)


def test_fetch_model_by_name(pkg):
    m = pkg.models.fetch_model_by_name("UNet", spatial_dims=3, in_channels=1, out_channels=2, channels=(16, 32, 64, 128, 256),
                                       strides=(2, 2, 2, 2), num_res_units=2, norm="INSTANCE")
    assert isinstance(m, pkg.UNet)


def test_monai_value_errors(pkg):
    with pytest.raises(ValueError):
        pkg.UNet(channels=(16,), strides=())
    with pytest.raises(ValueError):
        pkg.UNet(channels=(16, 32, 64), strides=(2,))
    m = pkg.UNet(channels=(16, 32), strides=(2, 2, 2))        # MONAI ignores the extra strides
    assert m.strides == [2]


@pytest.mark.parametrize("kw,word", [
    (dict(norm="BATCH"), "norm"), (dict(norm=("group", {"num_groups": 8})), "norm"),
    (dict(act=("prelu", {"num_parameters": 16})), "per-channel"), (dict(act="gelu"), "act"),
    (dict(dropout=0.1), "dropout"), (dict(adn_ordering="ADN"), "adn_ordering"),
    (dict(kernel_size=5), "kernel_size"), (dict(up_kernel_size=2), "up_kernel_size"),
    (dict(strides=(2, 1, 2, 2)), "strides"), (dict(spatial_dims=2), "spatial_dims"),
    (dict(channels=(12, 24, 48, 96, 192)), "channels"), (dict(out_channels=17), "out_channels"),
])
def test_unimplemented_options_raise(pkg, kw, word):
    with pytest.raises(NotImplementedError, match=word):
        pkg.UNet(**kw)


def test_plan_rejects_what_python_rejects(pkg):
    m = pkg.UNet(channels=(16, 32, 64), strides=(2, 2))
    with pytest.raises(RuntimeError, match="must be even"):
        _plan(pkg, m, 1, 34, 32, 32)   # 34 -> 17: not divisible by 2 ** len(strides)
    with pytest.raises(RuntimeError, match="act_kind"):
        _plan(pkg, m, 1, 32, 32, 32, act_kind=2)
    with pytest.raises(RuntimeError, match="out_channels"):
        _plan(pkg, m, 1, 32, 32, 32, n_outputs=17)


def test_tutorial_geometries_plan_within_40gb(pkg):
    spleen = pkg.UNet(in_channels=1, out_channels=2, channels=(16, 32, 64, 128, 256), strides=(2, 2, 2, 2), num_res_units=2)
    brats = pkg.UNet(in_channels=4, out_channels=3, channels=(16, 32, 64, 128, 256), strides=(2, 2, 2, 2), num_res_units=2)
    for m, shape in ((spleen, (4, 96, 96, 96)), (brats, (2, 128, 128, 128))):
        train = _plan(pkg, m, *shape)
        infer = _plan(pkg, m, *shape, inference_only=1)
        assert train.ws_bytes < 40 * 2 ** 30
        assert infer.ws_bytes < 0.6 * train.ws_bytes
