"""Host-only checks of the 256-voxel per-tap tile (k_igemm_conv_wide, no GPU needed): which launches of the C2, C3 and C5 plans
take it, and that the route query reports the geometry the launch runs.  tests/test_gpu_conv_wide_pair.py runs it against fp64
and bit for bit against the 128-voxel tile.

A per-tap launch at BN = 128 takes the 256-voxel tile (two consumer warpgroups) when its CTAs of that tile still give each of the
132 SMs one: N x ceil(D / 2 td) x (h, w tiles) x (N tiles) >= 132, with td the depth of the 128-voxel tile."""
import math

import pytest

import conv_route_cases as R
import plan_launches as P

SMS = 132
SMEM_LIMIT = 232448


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


def query(L, l, split, tile128=False):
    """conv_route_cases.conv_query of a plan launch, with the diagnostics option that keeps the 128-voxel tile"""
    sdims, ksz, stride, cls = R.conv_geometry(l.op, P.pad8(l.c), l.dims)
    x = R.ShapeAct(L, l.n, *sdims, P.pad8(l.c), split)
    out = R.ShapeAct(L, l.n, *l.dims, P.pad8(l.co), split)
    kw = dict(cls_mode=cls, mode=l.mode, ext=L.diag_ext(tile128=tile128))
    if l.c2:
        kw.update(x2=R.ShapeAct(L, l.n, *l.dims, P.pad8(l.c2), split), w2_hi=R.Addr(), w2_lo=R.Addr() if split else None,
                  cip2=P.pad8(l.c2))
    if l.mode == 1:
        kw.update(gn_x=R.ShapeAct(L, l.n, *l.dims, P.pad8(l.co), split), coef=R.Addr(), coef_ld=P.pad8(l.co), bstats=R.Addr())
    return L.conv3d_route(x, R.Addr(), R.Addr() if split else None, ksz, stride, out, P.pad8(l.co), P.pad8(l.c), **kw)


def conv_launches(config):
    return [l for l in P.BY_NAME[config].launches() if l.kernel in ("fwd", "dgrad")]


def expect_wide(l, narrow):
    """from the 128-voxel route of a launch: does the 256-voxel tile fill the GPU"""
    if narrow["kind"] != "tap" or narrow["bn"] != 128:
        return False
    d, h, w = l.dims
    tiles = l.n * math.ceil(d / (2 * narrow["td"])) * math.ceil(h / narrow["th"]) * math.ceil(w / narrow["tw"])
    return tiles * narrow["grid"][1] >= SMS


@pytest.mark.parametrize("config", ["C2", "C3", "C5"])
@pytest.mark.parametrize("split", [False, True], ids=["bf16", "split"])
def test_wide_tile_where_it_fills_the_gpu(L, config, split):
    wide = 0
    for l in conv_launches(config):
        r, narrow = query(L, l, split), query(L, l, split, tile128=True)
        assert narrow["wgs"] == (2 if narrow["kind"] == "pair" else 1)
        # the route table keys (kind, BN, KC, K chunks) do not depend on the tile
        assert (r["kind"], r["bn"], r["kc"], r["kchunks"], r["npass"]) == \
               (narrow["kind"], narrow["bn"], narrow["kc"], narrow["kchunks"], narrow["npass"]), (l, r, narrow)
        if not expect_wide(l, narrow):
            assert r == narrow, (config, l)
            continue
        wide += 1
        # the launch geometry: the 128-voxel tile doubled in depth, one CTA per 256-voxel tile and N tile
        assert r["wgs"] == 2 and (r["tw"], r["th"], r["td"]) == (narrow["tw"], narrow["th"], 2 * narrow["td"]), (l, r)
        d, h, w = l.dims
        assert r["grid"] == (l.n * math.ceil(d / r["td"]) * math.ceil(h / r["th"]) * math.ceil(w / r["tw"]), narrow["grid"][1], 1)
        assert r["grid"][0] * r["grid"][1] >= SMS
        assert r["blocks_per_sm"] == 1 and 3 <= r["stages"] <= 6 and r["smem_bytes"] <= SMEM_LIMIT
    assert wide > 0


def test_c2_wide_launches(L):
    """C2: the 128- and 256-channel launches at 32^3 and 64^3 take the 256-voxel tile; every launch at 16^3 (64 x 2 CTAs of the
    128-voxel tile) keeps the 128-voxel tile"""
    for l in conv_launches("C2"):
        for split in (False, True):
            r = query(L, l, split)
            if l.dims == (16, 16, 16):
                assert r["wgs"] == 1 and r["tw"] * r["th"] * r["td"] == 128, l
            elif r["kind"] == "tap" and r["bn"] == 128 and l.dims in ((32, 32, 32), (64, 64, 64)):
                assert r["wgs"] == 2 and (r["tw"], r["th"], r["td"]) == (8, 4, 8), l


def test_small_grids_keep_the_128_voxel_tile(L):
    """the per-tap cases of tests/conv_route_cases.py give fewer than 132 CTAs of 256 voxels"""
    for case in R.CONV_CASES + R.DEEP_K_CASES:
        r = R.conv_query(L, case.op, case.cin, case.cout, case.dims, case.split, case.mode, case.cin2)
        assert r["wgs"] == (2 if r["kind"] == "pair" else 1), case
