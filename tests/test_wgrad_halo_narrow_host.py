"""Host-only checks of the halo weight gradient (no GPU needed): the C2 layers at 128^3 take one 64-channel halo box per voxel tile
with the CTA shape of the two consumer warpgroups, inputs of up to 32 channels do so only at N tiles of at most 32 columns, and
what must stay on per-tap tiles (split precision, output planes smaller than the 8 x 16 halo tile, stride 2) does."""
import math

import pytest

import conv_route_cases as R


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


@pytest.mark.parametrize("ci,co,res,groups", [
    (8, 32, 128, 2),      # encoder conv1 (4 real input channels in an 8-channel view)
    (32, 32, 128, 2),     # encoder conv2, decoder conv2
    (64, 32, 128, 2),     # decoder conv1
    (16, 16, 128, 1),
    (64, 64, 64, 4),      # encoder level 1
    (40, 128, 32, 7),
])
@pytest.mark.parametrize("deterministic", [False, True])
def test_weight_gradients_take_halo_tiles(L, ci, co, res, groups, deterministic):
    r = R.wgrad_query(L, "k3s1", ci, co, (res, res, res), deterministic=deterministic)
    bn = R.kc_of(co) if co <= 64 else 128
    assert (r["kind"], r["cb"], r["bn"]) == ("halo", 64, bn)         # 64-channel box whatever the input's width
    qtiles = math.ceil(27 / 2)                                        # one tap per m64 half
    assert r["groups"] == groups == math.ceil(qtiles / (2 * (128 // bn)))   # two consumer warpgroups of 128 / BN M tiles each
    assert r["qt"] == math.ceil(qtiles / groups)
    assert (r["tw"], r["th"], r["td"]) == (8, 16, 1)
    kblocks = 2 * res * (res // 16) * (res // 8)
    assert r["kblocks"] == kblocks
    assert r["splits"] == min(kblocks, 132 // (groups * r["cotiles"]))
    assert r["part_bytes"] == r["splits"] * 27 * ci * co * 4


@pytest.mark.parametrize("ci", [8, 16, 24, 32])
@pytest.mark.parametrize("co", [40, 64, 128, 256])
def test_narrow_inputs_keep_per_tap_tiles_at_wide_n_tiles(L, ci, co):
    assert R.wgrad_query(L, "k3s1", ci, co, (64, 64, 64))["kind"] == "tap"


@pytest.mark.parametrize("ci", [8, 16, 24, 32, 40, 64])
def test_split_precision_small_planes_and_stride_two_stay_on_per_tap_tiles(L, ci):
    assert R.wgrad_query(L, "k3s1", ci, 32, R.LARGE_PLANE)["kind"] == "halo"
    assert R.wgrad_query(L, "k3s1", ci, 32, R.LARGE_PLANE, split=True)["kind"] == "tap"
    for dims in ((2, 15, 8), (2, 16, 7), R.SMALL_PLANE):
        assert R.wgrad_query(L, "k3s1", ci, 32, dims)["kind"] == "tap", dims
    assert R.wgrad_query(L, "k3s2", ci, 32, R.LARGE_PLANE)["kind"] == "tap"
