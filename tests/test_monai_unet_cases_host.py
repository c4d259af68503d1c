"""build_unet's launches as tests/monai_unet_cases.py restates them, held to the library: the MACs the plan counts, its parameter
spec, and a tensor-core route for every convolution of the benchmark workloads -- the transposed k3 s2 p1 output_padding 1
convolutions in all three directions and the stride-2 convolutions on the packed 8- or 16-channel input included -- the routes
of the spleen and BraTS workloads as monai_unet_cases.ROUTES / WGRAD_ROUTES table them, and the logits conv's per-tap route in
both precisions.  Host only."""
import dataclasses

import pytest
import torch

import monai_unet_cases as U
import plan_launches as PL


def _plan(pkg, config):
    desc = pkg.UNet(**config.kw)._net_desc(config.n, *config.dims)
    desc.inference_only = int(not config.train)
    desc.input_grad = int(config.input_grad)
    return pkg.models._Plan(desc, torch.device("cpu"))


@pytest.mark.parametrize("config", U.CONFIGS, ids=lambda c: c.name)
def test_restated_launches_are_the_plans(pkg, config):
    plan = _plan(pkg, config)
    launches = config.launches()
    macs = {k: float(sum(l.macs() for l in launches if l.kernel == k and not l.reads_input)) for k in ("fwd", "dgrad", "wgrad")}
    assert macs == {k: plan.algorithmic_macs()["conv_" + k] for k in macs}, config.name
    spec = plan.param_spec()
    assert sorted(l.key for l in launches if l.kernel == "fwd") == sorted(k for k, shape in spec if len(shape) == 5)
    norms = [l.key for l in launches if l.kernel == "gn"]
    assert len(set(norms)) == len(norms)
    for suffix in (".adn.N.weight", ".adn.A.weight"):   # affine norms and PReLU slopes belong to the restated norm-applies
        have = sorted(k[:-len(suffix)] for k, _ in spec if k.endswith(suffix))
        assert not have or have == sorted(norms), suffix


@pytest.mark.parametrize("split", [False, True], ids=["bf16", "split"])
@pytest.mark.parametrize("config", [c for c in U.CONFIGS if c.train], ids=lambda c: c.name)
def test_every_convolution_has_a_tensor_core_route(pkg, config, split):
    L = pkg.lib
    launches = config.launches()
    for l in launches:
        if l.kernel in ("fwd", "dgrad"):
            r = PL.conv_route(L, l, split)
            assert r["kind"] in L.CONV_KINDS and r["npass"] == (3 if split else 1), (l, r)
        elif l.kernel == "wgrad":
            assert PL.wgrad_route(L, l, split)["kind"] in L.WGRAD_KINDS, l
    convs = {(l.kernel, l.op, l.macs_div) for l in launches}
    # the transposed convolutions (LAYER_CONVT_OP1) in all three directions
    assert {("fwd", "k3s1", 8), ("wgrad", "k3s1", 8), ("dgrad", "k3s2", 1)} <= convs
    # the stride-2 convolutions on the packed input: forward and weight gradient, and the data gradient into it with input_grad
    first = [l for l in launches if l.key.startswith(("model.0.conv.", "model.0.residual."))]   # the top down layer
    cin = config.kw["in_channels"]
    assert any(l.kernel == "fwd" and l.op == "k3s2" and l.c == cin for l in first)
    assert any(l.kernel == "wgrad" and l.op == "k3s2" and l.c == cin for l in first)
    assert any(l.kernel == "dgrad" and l.reads_input and l.co == cin for l in launches) == config.input_grad


@pytest.mark.parametrize("split", [False, True], ids=["bf16", "split"])
@pytest.mark.parametrize("config", U.CONFIGS, ids=lambda c: c.name)
def test_the_logits_conv_runs_per_tap(pkg, config, split):
    """the conv that writes the logits stores its fp32 accumulators as hi + lo in both precisions (plan.cu: new_buf's force_lo):
    the halo kernels store hi only, so it runs on per-tap tiles where the same conv without the lo plane would take halo tiles"""
    L = pkg.lib
    top = "model.2.1.conv.unit0.conv.weight" if config.kw.get("num_res_units", 0) else "model.2.conv.weight"
    marked = [l for l in config.launches() if l.lo_out]
    assert [(l.kernel, l.key) for l in marked] == [("fwd", top)]
    assert PL.conv_route(L, marked[0], split)["kind"] == "tap"
    assert PL.conv_route(L, dataclasses.replace(marked[0], lo_out=False), False)["kind"] == "halo"


@pytest.mark.parametrize("split", [False, True], ids=["bf16", "split"])
@pytest.mark.parametrize("name", ["spleen", "brats"])
def test_benchmark_workloads_take_the_tabled_routes(pkg, name, split):
    """every convolution, data gradient and weight gradient of the two benchmark workloads on the route of
    monai_unet_cases.ROUTES / WGRAD_ROUTES (the host query assumes 132 SMs without a device)"""
    L = pkg.lib
    config = next(c for c in U.CONFIGS if c.name == name)
    precision = "split" if split else "bf16"
    assert U.route_table(L, config, split) == U.ROUTES[name][precision]
    assert U.wgrad_route_table(L, config, split) == U.WGRAD_ROUTES[name][precision]
