"""Host-only checks of the convolution and weight-gradient dispatch (no GPU needed): the route each launch takes, reported by the
library's route queries, is swept over the channel widths, extents, kernels, precisions and epilogues the plans use.  Every
reachable route must have a case in tests/conv_route_cases.py (which the GPU tests run against fp64 references), every
instantiated kernel must be reachable or listed with a reason, and the compile-time configurations behind the routes must keep
the occupancy and shared-memory rules the dispatch relies on."""
import math
import os
import re

import pytest

import conv_route_cases as R
import plan_launches as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "3dunetcnn_b200", "csrc")
SMEM_LIMIT = 232448          # sm_90 opt-in dynamic shared memory per block
SMEM_PER_SM = 233472         # 228 KB per SM; each resident block also reserves 1 KB


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


@pytest.fixture(scope="module")
def conv_sweep(L):
    return list(R.conv_sweep(L))


@pytest.fixture(scope="module")
def wgrad_sweep(L):
    return list(R.wgrad_sweep(L))


def _fmt(keys):
    return "\n  ".join(str(k) for k in sorted(keys))


def _macro_list(path, name):
    """the X(...) argument tuples of `#define name(X) ...` in a source file"""
    text = open(path).read()
    m = re.search(r"#define\s+%s\(X\)((?:[^\n]*\\\n)*[^\n]*)" % name, text)
    assert m, "%s not found in %s" % (name, path)
    return [tuple(int(v) for v in t.split(",")) for t in re.findall(r"X\(([\d,\s]+)\)", m.group(1))]


# ------------------------------------------------------------------------------------------------------------ convolution
def test_every_reachable_conv_route_has_a_case(conv_sweep):
    reachable = {R.route_key_of(p, r) for p, r in conv_sweep}
    table = [c.key for c in R.CONV_CASES]
    assert len(table) == len(set(table)), "duplicate cases for a route"
    missing = reachable - set(table)
    assert not missing, "convolution routes without a case in tests/conv_route_cases.py:\n  " + _fmt(missing)
    stale = set(table) - reachable
    assert not stale, "cases for routes the sweep no longer reaches:\n  " + _fmt(stale)


@pytest.mark.parametrize("case", R.CONV_CASES, ids=lambda c: c.id)
def test_conv_case_takes_its_route(L, case):
    r = R.conv_query(L, case.op, case.cin, case.cout, case.dims, case.split, case.mode, case.cin2)
    assert r is not None, "the library refuses the case"
    assert (r["kind"], r["bn"], r["kc"]) == (case.kind, case.bn, case.kc)
    assert r["kchunks"] == case.kchunks
    assert r["npass"] == (3 if case.split else 1)
    assert r["cls_pair"] == int(case.kind.startswith("class") and not case.split)
    # grid: one CTA per (sample, voxel tile) and N tile
    gdims = case.dims if not case.kind.startswith("class") else tuple(v // 2 for v in case.dims)
    tiles = math.ceil(gdims[0] / r["td"]) * math.ceil(gdims[1] / r["th"]) * math.ceil(gdims[2] / r["tw"])
    assert r["grid"] == (2 * tiles, math.ceil(case.cout / case.bn), 1)
    assert r["tw"] * r["th"] * r["td"] == 128
    # the case exercises partial tiles: the last N tile and at least one spatial axis
    if case.bn > 16:
        assert case.cout % case.bn != 0 or case.kind.startswith("class")
    assert any(g % t for g, t in zip(gdims, (r["td"], r["th"], r["tw"])))


def test_kc64_cases_walk_several_k_chunks_in_every_kind():
    kinds = {c.kind for c in R.CONV_CASES if c.kc == 64 and c.kchunks[0] > 1}
    assert kinds == {"tap", "class1", "class2"}           # halo mode loads one K chunk of its 3x3x3 source
    assert any(c.kind == "halo" and c.nsrc == 2 and c.kchunks[1] > 1 for c in R.CONV_CASES), "wide second source in halo mode"
    assert any(c.kind == "tap" and c.nsrc == 2 and c.kchunks[1] > 1 for c in R.CONV_CASES), "wide second source on per-tap tiles"
    assert any(c.kind == "halo" and c.mode == 1 and c.bn <= 32 for c in R.CONV_CASES), "mode 1 on the halo kernel at BN <= 32"


@pytest.mark.parametrize("case", R.DEEP_K_CASES, ids=R.deep_k_id)
def test_deep_k_case_takes_its_route(L, case):
    r = R.conv_query(L, case.op, case.cin, case.cout, case.dims, case.split, case.mode, case.cin2)
    assert (r["kind"], r["bn"], r["kc"], r["kchunks"]) == (case.kind, case.bn, case.kc, case.kchunks)
    assert r["npass"] == (3 if case.split else 1)
    assert case.key in {c.key for c in R.CONV_CASES}, "a deep-K case of a route without a case in CONV_CASES"


# the configurations of tests/plan_launches.py whose K loops need fp64 cases: the benchmark's C2 and C3 training steps and C5
# forward, the BraTS DynUNet and the SegResNet recipes
DEEP_K_CONFIGS = ["C2", "C3", "C5", "brats-dynunet", "brats-segresnet"] + [c.name for c in P.CONFIGS
                                                                          if c.name.startswith("segresnet-")]


def test_deep_k_loops_of_the_restated_configurations_have_fp64_cases(L):
    """for each (kind, KC, precision, mode) the largest K-chunk count, per source, that a layer of the DEEP_K_CONFIGS walks in
    either precision must be walked by a case the GPU tests run against fp64 (CONV_CASES + DEEP_K_CASES)"""
    have = {}
    for c in R.CONV_CASES + R.DEEP_K_CASES:
        k = (c.kind, c.kc, "split" if c.split else "bf16", c.mode)
        have[k] = tuple(max(a, b) for a, b in zip(have.get(k, (0, 0)), c.kchunks))
    need = {}
    for config in DEEP_K_CONFIGS:
        for l in P.BY_NAME[config].launches():
            if l.kernel not in ("fwd", "dgrad"):
                continue
            for split in (False, True):
                r = P.conv_route(L, l, split)
                assert r is not None, (config, l, split)
                k = (r["kind"], r["kc"], "split" if split else "bf16", l.mode)
                for s in (0, 1):
                    if r["kchunks"][s] > need.get((k, s), (1, None))[0]:
                        need[(k, s)] = (r["kchunks"][s], "%s %s %s" % (config, l.kernel, l.key))
    assert max(v[0] for v in need.values()) == 12          # the C5 network's 768-channel layers
    short = ["%s source %d: %d K chunks (%s), the cases walk %d" % (k, s, m, where, have.get(k, (0, 0))[s])
             for (k, s), (m, where) in sorted(need.items()) if have.get(k, (0, 0))[s] < m]
    assert not short, "K loops deeper than any fp64 case walks:\n  " + "\n  ".join(short)


def test_c5_routes(L):
    import c5_cases
    for precision in ("bf16", "split"):
        assert c5_cases.route_table(L, precision == "split") == c5_cases.C5_ROUTES[precision]


def test_instantiated_conv_kernels_are_reachable_or_listed(conv_sweep):
    configs = _macro_list(os.path.join(CSRC, "igemm_conv.cu"), "B200_CONV_CONFIGS")
    assert len(configs) >= 12
    reached = {(r["kind"], r["bn"], r["kc"]) for _, r in conv_sweep}
    for kind in ("tap", "halo", "class1", "class2"):
        for bn, kc in configs:
            k = (kind, bn, kc)
            if k in R.CONV_UNREACHABLE:
                assert k not in reached, "%s is reachable now: remove it from CONV_UNREACHABLE and add its cases" % (k,)
            else:
                assert k in reached, "%s is instantiated but no launch of the sweep reaches it: add a case or list why" % (k,)
    assert set(R.CONV_UNREACHABLE) <= {(kind, bn, kc) for kind in ("tap", "halo", "class1", "class2") for bn, kc in configs}


def test_halo_mode_never_costs_occupancy(L, conv_sweep):
    """halo tiles must keep at least the CTAs per SM of per-tap tiles for the same (BN, KC); the per-tap numbers come from the
    same channels on a plane too small for halo tiles"""
    checked = 0
    for p, r in conv_sweep:
        if r["kind"] != "halo":
            continue
        tap = R.conv_query(L, "k3s1", p["cin"], p["cout"], R.SMALL_PLANE, p["split"], p["mode"], p["cin2"])
        assert tap["kind"] == "tap" and (tap["bn"], tap["kc"]) == (r["bn"], r["kc"])
        assert r["blocks_per_sm"] >= tap["blocks_per_sm"], (p, r["blocks_per_sm"], tap["blocks_per_sm"])
        checked += 1
    assert checked > 0


def test_halo_mode_reads_one_k_chunk_of_its_3x3x3_source(L, conv_sweep):
    """the halo box holds one K chunk: every halo route of the sweep has kchunks[0] == 1, and a 3x3x3 source wider than 64
    channels on a plane that fills the halo tile runs on per-tap tiles in both precisions"""
    halo = [(p, r) for p, r in conv_sweep if r["kind"] == "halo"]
    assert halo
    for p, r in halo:
        assert r["kchunks"][0] == 1, (p, r)
    for cin in (72, 128, 256):
        for split in (False, True):
            r = R.conv_query(L, "k3s1", cin, 64, R.LARGE_PLANE, split)
            assert r["kind"] == "tap" and r["kchunks"][0] > 1, (cin, split, r)


def test_conv_configurations_fit_shared_memory(conv_sweep):
    seen = {}
    for _, r in conv_sweep:
        seen[(r["kind"], r["bn"], r["kc"])] = (r["stages"], r["blocks_per_sm"], r["smem_bytes"])
    for k, (stages, bps, smem) in seen.items():
        assert 2 <= stages <= 6, k
        assert smem <= SMEM_LIMIT, k
        assert bps in (1, 2), k
        if bps == 2:
            assert 2 * (smem + 1024) <= SMEM_PER_SM, k


def test_k_chunk_follows_the_widest_source_with_the_largest_kernel(conv_sweep):
    for p, r in conv_sweep:
        ksz0 = R.conv_geometry(p["op"], p["cin"], p["dims"])[1]
        if p["cin2"] and ksz0 == 1:          # both 1x1x1: the wider one
            c = max(p["cin"], p["cin2"])
        else:                                # the 3x3x3 (or 2x2x2) first source, however wide the 1x1x1 second one is
            c = p["cin"]
        assert r["kc"] == R.kc_of(c), p
        assert r["kchunks"] == (math.ceil(p["cin"] / r["kc"]), math.ceil(p["cin2"] / r["kc"]) if p["cin2"] else 0), p


def test_route_query_refuses_what_the_launcher_refuses(L):
    assert R.conv_query(L, "class1", 32, 32, (4, 6, 8), mode=1) is None          # class mode: plain epilogue only
    assert R.conv_query(L, "k3s1", 12, 32, R.SMALL_PLANE) is None                 # channels: multiples of 8
    with pytest.raises(RuntimeError, match="split mode needs a lo output"):
        x = R.ShapeAct(L, 2, *R.SMALL_PLANE, 16, split=True)
        L.conv3d_route(x, R.Addr(), R.Addr(), 3, 1, R.ShapeAct(L, 2, *R.SMALL_PLANE, 16), 16, 16)


# ------------------------------------------------------------------------------------------------------- weight gradient
def test_every_reachable_wgrad_route_has_a_case(wgrad_sweep):
    reachable = {R.wgrad_route_key(p["split"], r) for p, r in wgrad_sweep}
    table = [c.key for c in R.WGRAD_CASES]
    assert len(table) == len(set(table)), "duplicate cases for a route"
    missing = reachable - set(table)
    assert not missing, "weight-gradient routes without a case in tests/conv_route_cases.py:\n  " + _fmt(missing)
    stale = set(table) - reachable
    assert not stale, "cases for routes the sweep no longer reaches:\n  " + _fmt(stale)


@pytest.mark.parametrize("case", R.WGRAD_CASES, ids=lambda c: c.id)
def test_wgrad_case_takes_its_route(L, case):
    r = R.wgrad_query(L, case.op, case.ci, case.co, case.dims, case.split)
    assert r is not None
    assert R.wgrad_route_key(case.split, r) == case.key
    det = R.wgrad_query(L, case.op, case.ci, case.co, case.dims, case.split, deterministic=True)
    assert det["kind"] in ("tap", "halo")                  # the SIMT kernel only accumulates with atomics
    if case.kind != "simt":
        assert det == r
        assert r["npass"] == (3 if case.split else 1)
        assert r["cotiles"] == math.ceil(case.co / case.bn)


def test_instantiated_wgrad_kernels_are_reachable_or_listed(wgrad_sweep):
    src = os.path.join(CSRC, "wgrad.cu")
    tap = [("tap", cb, bn) for cb, bn in _macro_list(src, "B200_WG_CONFIGS")]
    halo = [("halo", 64, bn) for (bn,) in _macro_list(src, "B200_WG_HALO_CONFIGS")]
    assert len(tap) == 12 and len(halo) == 4
    reached = {(r["kind"], r["cb"], r["bn"]) for _, r in wgrad_sweep if r["kind"] != "simt"}
    for k in tap + halo:
        if k in R.WGRAD_UNREACHABLE:
            assert k not in reached, "%s is reachable now: remove it from WGRAD_UNREACHABLE and add its cases" % (k,)
        else:
            assert k in reached, "%s is instantiated but no launch of the sweep reaches it: add a case or list why" % (k,)
    simt = {r["ci8"] for _, r in wgrad_sweep if r["kind"] == "simt"}
    assert simt == {1, 2}


def test_wgrad_partial_bytes_cover_both_tilings(L):
    """the plans size the deterministic partial buffer with wgrad_partial_bytes from shapes alone, before they know whether a
    launch runs in bf16 (halo tiles possible) or split precision (per-tap tiles): it must cover the route of either"""
    for op in ("k3s1", "k3s2", "k1", "k2s2"):
        for dims in (R.SMALL_PLANE, R.LARGE_PLANE, (1, 16, 8)):
            for ci in R.CHANNELS:
                for co in R.CHANNELS:
                    for sms in (132, 114):
                        adims, ksz, stride = R.wgrad_geometry(op, dims)
                        a, dy = R.ShapeAct(L, 2, *adims, ci), R.ShapeAct(L, 2, *dims, co)
                        have = L.wgrad_partial_bytes(a, dy, ksz, stride, ci, co, num_sms=sms)
                        for split in (False, True):
                            r = R.wgrad_query(L, op, ci, co, dims, split, deterministic=True, num_sms=sms)
                            assert r["part_bytes"] == r["splits"] * ksz ** 3 * ci * co * 4
                            assert have >= r["part_bytes"], (op, dims, ci, co, split, sms)
