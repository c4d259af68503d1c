"""The plan launches restated in tests/plan_launches.py, which the host tests derive their GPU cases from, held to the library
for every configuration of its catalogue.  Host only: creating a plan is bookkeeping."""
import pytest
import torch

import plan_launches as P


@pytest.mark.parametrize("config", P.CONFIGS, ids=lambda c: c.name)
def test_restated_launches_are_the_plans(pkg, config):
    """the restated convolutions carry exactly the MACs the plan counts, forward, data gradient and weight gradient (plan.cu:
    conv_macs; the packed input's padding channels carry none, and a data gradient into the network input is not counted), and
    the conv and head weights of the forward launches and the norms of the gn launches are the plan's parameter spec, each
    restated once"""
    desc = getattr(pkg, config.arch)(**config.kw)._net_desc(config.n, *config.dims)
    desc.inference_only = int(not config.train)
    desc.input_grad = int(config.input_grad)
    plan = pkg.models._Plan(desc, torch.device("cpu"))
    launches = config.launches()
    macs = {k: float(sum(l.macs() for l in launches if l.kernel == k and not l.reads_input)) for k in ("fwd", "dgrad", "wgrad")}
    assert macs == {k: plan.algorithmic_macs()["conv_" + k] for k in macs}, config.name
    spec = plan.param_spec()
    weights = [l.key for l in launches if l.kernel in ("fwd", "head_fwd")] + [l.key2 for l in launches if l.key2]
    assert sorted(weights) == sorted(k for k, shape in spec if len(shape) == 5), config.name
    norms = [l.key for l in launches if l.kernel == "gn"]
    assert sorted(norms) == sorted(k[:-len(".weight")] for k, shape in spec
                                   if len(shape) == 1 and k.endswith(".weight")), config.name
