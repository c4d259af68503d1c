"""Host-only checks of the (BN 64, KC 64) halo convolutions on the weight-only ring (no GPU needed): every such launch of the
benchmark and recipe plans keeps its route and launch geometry (one consumer warpgroup, one CTA per 8 x 16 x 1 tile) and runs
two CTAs per SM.  tests/test_gpu_conv_halo_ring2.py runs the kernel against fp64 and bit for bit against per-tap tiles."""
import math

import pytest

import plan_launches as P

TWO_PER_SM = 115712          # half of the SM's 228 KB, less the 1 KB the hardware reserves per CTA
# launches per plan (forward and data gradient): C2 / C3 encoder level 1 at 64^3, C5's two at 128^3 with a fused 1x1x1 source
EXPECTED = {"C2": 6, "C3": 6, "C5": 2, "brats-dynunet": 4, "brats-segresnet": 12}


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


def ring_launches(L, config):
    """(launch, route) of every bf16 forward / data-gradient launch of config on the (halo, 64, 64) route"""
    out = []
    for l in P.BY_NAME[config].launches():
        if l.kernel not in ("fwd", "dgrad"):
            continue
        r = P.conv_route(L, l, False)
        if (r["kind"], r["bn"], r["kc"]) == ("halo", 64, 64):
            out.append((l, r))
    return out


@pytest.mark.parametrize("config", [c.name for c in P.CONFIGS])
def test_ring_halo_launches_run_two_ctas_per_sm(L, config):
    launches = ring_launches(L, config)
    if config in EXPECTED:
        assert len(launches) == EXPECTED[config], [l for l, _ in launches]
    for l, r in launches:
        d, h, w = l.dims
        assert r["kchunks"] == (1, math.ceil(P.pad8(l.c2) / 64)) and r["npass"] == 1, (l, r)
        assert r["wgs"] == 1 and (r["tw"], r["th"], r["td"]) == (8, 16, 1), (l, r)
        assert r["grid"] == (l.n * d * math.ceil(h / 16) * math.ceil(w / 8), math.ceil(P.pad8(l.co) / 64), 1), (l, r)
        assert r["blocks_per_sm"] == 2 and r["stages"] == 4 and r["smem_bytes"] <= TWO_PER_SM, (l, r)


def test_c5_fused_sources(L):
    """C5's two launches read a fused 1x1x1 source in one and in two K chunks (+8 and +96 channels)"""
    assert sorted(r["kchunks"] for _, r in ring_launches(L, "C5")) == [(1, 1), (1, 2)]
