"""Host-only checks of the two-plane halo route (no GPU needed): which launches take it, and the compile-time configuration it
reports.  tests/test_gpu_conv_halo_pair.py runs it against fp64 and bit for bit against per-tap tiles."""
import math

import pytest

import conv_route_cases as R

SMEM_LIMIT = 232448          # sm_90 opt-in dynamic shared memory per block
BIG = (128, 128, 128)


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


@pytest.mark.parametrize("cin,cout,mode,bn,kc", [(64, 32, 0, 32, 64), (64, 32, 1, 32, 64), (32, 64, 0, 64, 32), (32, 64, 1, 64, 32),
                                                 (40, 24, 0, 32, 64), (24, 40, 1, 64, 32)])
def test_full_size_single_source_launches_take_the_pair_route(L, cin, cout, mode, bn, kc):
    r = R.conv_query(L, "k3s1", cin, cout, BIG, mode=mode)
    assert (r["kind"], r["bn"], r["kc"], r["kchunks"], r["npass"]) == ("pair", bn, kc, (1, 0), 1), r
    assert (r["tw"], r["th"], r["td"]) == (8, 16, 1)
    assert (r["stages"], r["blocks_per_sm"]) == (2, 1)
    assert r["smem_bytes"] <= SMEM_LIMIT
    units = 2 * math.ceil(BIG[0] / 2) * (BIG[1] // 16) * (BIG[2] // 8)
    assert 1 <= r["grid"][0] <= units and r["grid"][1:] == (1, 1)      # persistent: one CTA per SM at most


def test_other_launches_keep_their_routes(L):
    # below one unit per SM the tiles stay on the per-tile kernels: 2 x 2 x 2 x 2 = 16 units
    assert (R.conv_query(L, "k3s1", 64, 32, R.H)["kind"], R.conv_query(L, "k3s1", 32, 64, R.H)["kind"]) == ("tap", "halo")
    # split precision, a fused 1x1x1 second source, stride 2 and other (BN, KC) keep theirs at full size too
    assert R.conv_query(L, "k3s1", 64, 32, BIG, split=True)["kind"] == "tap"
    assert R.conv_query(L, "k3s1", 32, 64, BIG, cin2=16)["kind"] == "halo"
    assert R.conv_query(L, "k3s1", 64, 32, BIG, cin2=16)["kind"] == "tap"
    assert R.conv_query(L, "k3s2", 64, 32, (64, 64, 64))["kind"] == "tap"
    for cin, cout in ((32, 32), (64, 64), (8, 32), (32, 8)):
        assert R.conv_query(L, "k3s1", cin, cout, BIG)["kind"] == "halo", (cin, cout)
