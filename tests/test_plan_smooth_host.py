"""The smooth plan rows (tests/plan_smooth_cases.py) on the CPU: each row's fp64 noise floor leaves its bound room for the
plan's own rounding, the real activations would not, the rows together reach every wiring path of the two plan builders,
and the plan accepts every row.  Host only: the fp64 oracle and the host-side plan construction."""
import collections
import ctypes as C

import pytest

import plan_smooth_cases as P


@pytest.mark.parametrize("case", P.CASES, ids=lambda c: c.id)
def test_noise_floor_is_within_the_bound(case):
    b = P.BOUNDS[case.precision]
    floor = P.noise_floor(case, b["floor_eps"])
    over = {k: (v, P.bound_of(k, case.precision)) for k, v in floor.items() if v > P.bound_of(k, case.precision) / b["floor_div"]}
    assert not over, "noise floor at eps %g above bound / %g: %r" % (b["floor_eps"], b["floor_div"], over)


@pytest.mark.parametrize("arch", ["unet3d", "dynunet"])
def test_real_activation_floor_exceeds_the_split_bound(arch):
    """why the rows run at slope 1: with ReLU / LeakyReLU(0.01) the fp64 reference itself moves by more than the bound"""
    case = P.first(arch)
    floor = P.noise_floor(case, P.BOUNDS["split"]["floor_eps"], slope=P.real_slope(case))
    assert any(v > P.bound_of(k, "split") for k, v in floor.items()), floor


def test_rows_cover_every_wiring_path():
    have = set().union(*(P.features(c) for c in P.CASES))
    assert not P.REQUIRED_FEATURES - have, sorted(P.REQUIRED_FEATURES - have)


def test_rows_are_well_formed():
    assert max(collections.Counter(c.id for c in P.CASES).values()) == 1
    for case in P.CASES:
        _, _, _, mask = P.inputs(case)
        if case.arch == "unet3d" and case.train:
            assert bool((mask == 0).any(dim=1).all()) and bool((mask > 0).any()), case.id
        else:
            assert mask is None, case.id
        assert case.train or case.arch == "unet3d"           # the DynUNet plan has no in-model activation


@pytest.mark.parametrize("case", P.CASES, ids=lambda c: c.id)
def test_plan_accepts_the_row(pkg, case):
    L = pkg.lib
    lib = L.load_library()
    model = P.model_of(pkg, case)
    n, _, d, h, w = case.shape
    desc = model._net_desc(n, d, h, w)
    assert desc.act_slope == P.SMOOTH
    desc.inference_only = int(not case.train)
    desc.input_grad = int(case.input_grad)
    desc.deterministic = int(case.deterministic)
    handle = C.c_void_p()
    L.check(lib.b200unet_plan_create(C.byref(desc), C.byref(handle)), "plan_create " + case.id)
    lib.b200unet_plan_destroy(handle)
