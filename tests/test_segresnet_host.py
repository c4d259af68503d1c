"""Host logic of the SegResNet mirror (no GPU): MONAI kwarg surface, state-dict spec == the restated oracle spec == the library
plan's spec, loud rejection of what is not implemented, the oracle against a module restatement, and the split-plan bounds of
tests/test_gpu_segresnet.py against the fp64 noise floor."""
import pytest
import torch
from torch import nn

import segresnet_cases as S
from oracle.segresnet_oracle import make_segresnet_state_dict, segresnet_forward, segresnet_state_dict_spec

CPU = torch.device("cpu")
SPEC_KW = [dict(), S.BRATS, dict(S.THREE_LEVEL)]


def _plan(pkg, m, n=1, dims=(32, 32, 32), **flags):
    d = m._net_desc(n, *dims)
    for k, v in flags.items():
        setattr(d, k, v)
    return pkg.models._Plan(d, CPU)


@pytest.mark.parametrize("kw", SPEC_KW, ids=["monai_defaults", "brats_recipe", "three_level"])
def test_state_dict_and_plan_spec(pkg, kw):
    m = pkg.SegResNet(**kw)
    spec = segresnet_state_dict_spec(**S.spec_kw(kw))
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == spec
    dims = (24, 32, 40) if len(S.spec_kw(kw)["blocks_down"]) == 3 else (32, 32, 32)
    plan = _plan(pkg, m, dims=dims)
    assert plan.param_spec() == spec
    assert _plan(pkg, m, dims=dims, inference_only=1).ws_bytes < 0.5 * plan.ws_bytes
    assert _plan(pkg, m, dims=dims, input_grad=1, deterministic=1, split_precision=1).param_spec() == spec
    m.load_state_dict(make_segresnet_state_dict(**S.spec_kw(kw)), strict=True)


def test_npow2_case_plan_spec(pkg):
    """the non-power-of-two case of the GPU tests: its plan builds at the case's shape with the oracle's spec, 12 input channels
    packed into 16"""
    case = S.NPOW2_CASE
    m = pkg.SegResNet(**case.kw)
    spec = segresnet_state_dict_spec(**S.spec_kw(case.kw))
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == spec
    assert (m.num_groups, m.dropout_width) == (8, 24)
    assert _plan(pkg, m, case.shape[0], case.shape[2:]).param_spec() == spec


def test_monai_defaults_and_init(pkg):
    m = pkg.SegResNet()
    assert (m.init_filters, m.in_channels, m.out_channels, m.blocks_down, m.blocks_up, m.num_groups) == (8, 1, 2, [1, 2, 2, 4], [1, 1, 1], 8)
    assert m.act_slope == 0.0 and m.dropout_p == 0.0
    sd = m.state_dict()
    assert torch.equal(sd["down_layers.0.1.norm1.weight"], torch.ones(8)) and torch.equal(sd["conv_final.0.bias"], torch.zeros(8))
    w = sd["down_layers.1.0.conv.weight"]                         # torch default: U(+-1/sqrt(fan_in)), fan_in = 8 * 27
    assert float(w.abs().max()) <= (8 * 27) ** -0.5 and float(w.std()) > 0.5 * (8 * 27) ** -0.5 / 3 ** 0.5


@pytest.mark.parametrize("kw,slope,groups", [
    (dict(act="relu"), 0.0, 8), (dict(act="RELU"), 0.0, 8), (dict(act=("leakyrelu", {"negative_slope": 0.2})), 0.2, 8),
    (dict(act=["LEAKYRELU", {"inplace": True}]), 0.01, 8), (dict(act="leakyrelu"), 0.01, 8),
    (dict(norm="group"), 0.0, 8), (dict(norm=["GROUP", {"num_groups": 4}]), 0.0, 4), (dict(norm_name="group", num_groups=2), 0.0, 2),
    (dict(norm=("group", {"num_groups": 8, "eps": 1e-5, "affine": True})), 0.0, 8),
])
def test_kwarg_spellings(pkg, kw, slope, groups):
    m = pkg.SegResNet(blocks_down=[1, 2, 2, 4], blocks_up=(1, 1, 1), **kw)
    assert m.act_slope == pytest.approx(slope) and m.num_groups == groups
    assert _plan(pkg, m).n_params == len(m.state_dict())


def test_fetch_model_by_name_json_block(pkg):
    block = {"name": "SegResNet", "init_filters": 16, "in_channels": 4, "out_channels": 3, "dropout_prob": 0.2,
             "blocks_down": [1, 2, 2, 4], "blocks_up": [1, 1, 1], "act": ["RELU", {"inplace": True}], "norm": ["GROUP", {"num_groups": 8}]}
    name = block.pop("name")
    m = pkg.fetch_model_by_name(name, **block)
    assert isinstance(m, pkg.SegResNet) and m.dropout_p == 0.2 and m.dropout_width == 16
    assert _plan(pkg, m, 1, (224, 224, 144)).ws_bytes < 20 * 2 ** 30


@pytest.mark.parametrize("bad", [dict(upsample_mode="deconv"), dict(upsample_mode="pixelshuffle"), dict(use_conv_final=False),
                                 dict(spatial_dims=2), dict(norm=("batch", {})), dict(norm="instance"), dict(norm_name="batch"),
                                 dict(act="prelu"), dict(act=("elu", {})), dict(blocks_down=(1, 0, 2, 4)), dict(blocks_up=(1, 0, 1)),
                                 dict(blocks_up=(1, 1)), dict(blocks_down=(1, 2), blocks_up=(1, 1))])
def test_unimplemented_options_raise(pkg, bad):
    with pytest.raises(NotImplementedError):
        pkg.SegResNet(**bad)


@pytest.mark.parametrize("kw", [dict(init_filters=8, num_groups=3, norm=("group", {"num_groups": 3})), dict(norm_name="group", num_groups=16),
                                dict(init_filters=24, norm=("group", {"num_groups": 16}))])
def test_groups_not_dividing_init_filters_raise_value_error(pkg, kw):
    with pytest.raises(ValueError):
        pkg.SegResNet(**kw)


def test_plan_rejections(pkg):
    with pytest.raises(RuntimeError, match=r"status -2\).*multiple of 8"):
        _plan(pkg, pkg.SegResNet(init_filters=12, norm=("group", {"num_groups": 4})))
    with pytest.raises(RuntimeError, match=r"status -2\).*must be even"):
        _plan(pkg, pkg.SegResNet(), dims=(36, 32, 32))            # 36 -> 18 -> 9: odd before the last level
    with pytest.raises(RuntimeError, match=r"status -2\).*64 channels into the head"):
        _plan(pkg, pkg.SegResNet(init_filters=128, out_channels=9, blocks_down=(1, 1), blocks_up=(1,)), dims=(8, 8, 8))
    assert _plan(pkg, pkg.SegResNet(init_filters=64, out_channels=9, blocks_down=(1, 1), blocks_up=(1,)), dims=(8, 8, 8)).n_params
    with pytest.raises(RuntimeError, match=r"status -2\).*1024"):
        _plan(pkg, pkg.SegResNet(init_filters=256, blocks_down=(1, 1, 1, 1), blocks_up=(1, 1, 1)), dims=(16, 16, 16))


# ------------------------------------------------------------------------------------------------ the oracle itself
class _ResBlock(nn.Module):
    def __init__(self, c, g, slope):
        super().__init__()
        self.norm1, self.norm2 = nn.GroupNorm(g, c), nn.GroupNorm(g, c)
        self.act = nn.LeakyReLU(slope) if slope else nn.ReLU()
        self.conv1 = nn.Sequential()
        self.conv1.add_module("conv", nn.Conv3d(c, c, 3, padding=1, bias=False))
        self.conv2 = nn.Sequential()
        self.conv2.add_module("conv", nn.Conv3d(c, c, 3, padding=1, bias=False))

    def forward(self, x):
        return self.conv2(self.act(self.norm2(self.conv1(self.act(self.norm1(x)))))) + x


def _conv(ci, co, k=3, s=1, bias=False):
    m = nn.Sequential()
    m.add_module("conv", nn.Conv3d(ci, co, k, stride=s, padding=k // 2, bias=bias))
    return m


class _ModuleSegResNet(nn.Module):
    """a second restatement from nn modules, registered in MONAI's order"""

    def __init__(self, cin, cout, f, bd, bu, g, slope):
        super().__init__()
        L = len(bd)
        self.convInit = _conv(cin, f)
        self.down_layers = nn.ModuleList(
            nn.Sequential(_conv(f << (i - 1), f << i, s=2) if i else nn.Identity(), *[_ResBlock(f << i, g, slope) for _ in range(n)])
            for i, n in enumerate(bd))
        self.up_layers = nn.ModuleList(nn.Sequential(*[_ResBlock(f << (L - 2 - i), g, slope) for _ in range(n)]) for i, n in enumerate(bu))
        self.up_samples = nn.ModuleList(
            nn.Sequential(_conv(f << (L - 1 - i), f << (L - 2 - i), k=1), nn.Upsample(scale_factor=2, mode="trilinear", align_corners=False))
            for i in range(L - 1))
        self.conv_final = nn.Sequential(nn.GroupNorm(g, f), nn.LeakyReLU(slope) if slope else nn.ReLU(), _conv(f, cout, k=1, bias=True))

    def forward(self, x, scale=None):
        x = self.convInit(x)
        if scale is not None:
            x = x * scale[:, :, None, None, None]
        down_x = []
        for d in self.down_layers:
            x = d(x)
            down_x.append(x)
        down_x.reverse()
        for i, (up, upl) in enumerate(zip(self.up_samples, self.up_layers)):
            x = upl(up(x) + down_x[i + 1])
        return self.conv_final(x)


@pytest.mark.parametrize("case", S.RELU_CASES + [S.SMOOTH_CASE], ids=lambda c: c.id)
def test_oracle_matches_module_restatement(case):
    sd, x, _, scale = S.inputs(case)
    kw = S.spec_kw(case.kw)
    bd, bu = case.blocks
    net = _ModuleSegResNet(kw["in_channels"], kw["out_channels"], kw["init_filters"], bd, bu, case.groups, S.slope_of(case.kw)).double()
    assert [(k, tuple(v.shape)) for k, v in net.state_dict().items()] == segresnet_state_dict_spec(**kw)
    net.load_state_dict({k: v.double() for k, v in sd.items()}, strict=True)
    with torch.no_grad():
        ref = net(x.double(), scale.double() if scale is not None else None)
        got = segresnet_forward({k: v.double() for k, v in sd.items()}, x.double(), bd, bu, case.groups, scale, S.slope_of(case.kw))
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-12


# ------------------------------------------------------------------------------------------------ bounds from the noise floor
def test_smooth_split_bounds_sit_above_the_noise_floor():
    b = S.SMOOTH_BOUNDS
    floor = S.noise_floor(S.SMOOTH_CASE, b["floor_eps"])
    for k, v in floor.items():
        bound = b["logits"] if k in ("logits", "loss") else b["grad"]
        assert v <= bound / b["floor_div"], (k, v, bound)


def test_relu_split_bounds_sit_above_the_noise_floor():
    """the 1e-3 logits bar of the ReLU cases holds 4x above the split-storage floor of every case"""
    for case in S.RELU_CASES:
        floor = S.noise_floor(case, S.SMOOTH_BOUNDS["floor_eps"], runs=1, input_grad=False)
        assert floor["logits"] <= S.RELU_BOUNDS["logits"] / 4 and floor["loss"] <= S.RELU_BOUNDS["loss"] / 4, (case.id, floor["logits"])


def _bf16_floor_below_bounds(case):
    floor = S.noise_floor(case, 2.0 ** -8, runs=1, input_grad=False)
    assert floor["loss"] * float(S.reference(case)["loss"]) <= S.BF16_DICE
    assert floor["logits"] <= S.BF16_LOGITS


def test_bf16_dice_bound_sits_above_the_noise_floor():
    """bf16 storage (eps 2^-8) moves the sigmoid Dice of the bf16 case by less than its bound"""
    _bf16_floor_below_bounds(S.RELU_CASES[1])


def test_npow2_bf16_dice_bound_sits_above_the_noise_floor():
    """the same for the non-power-of-two widths of tests/test_gpu_segresnet.py's second bf16 run"""
    _bf16_floor_below_bounds(S.NPOW2_CASE)
