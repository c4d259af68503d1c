"""The two-plane halo kernel (k_igemm_conv_halo_pair): (BN, KC) = (32, 64) and (64, 32), one source, from one unit of two
output planes per SM upward.

- Against fp64, as tests/test_gpu_conv_routes.py bounds the routes, on the odd-extent halo plane with an odd depth of 33: 17
  units per sample, the last one with its second plane outside the volume, a partial last N tile, and (mode 0) a CTA cap that
  makes every CTA walk several units across the sample boundary.
- At the C2 shapes (batch 2, 128^3): the 64 -> 32 forward and the 32 -> 64 mode-1 data gradient store the same bits as the same
  op on per-tap tiles (B200UNET_NO_HALO=1, in a child process): with one K chunk both accumulate every output row in the same
  order.  The per-channel statistics sum other fp32 per-tile partials (128-voxel tiles of another shape), so they agree to fp32
  rounding only."""
import os
import subprocess
import sys
import zlib

import pytest
import torch

import conv_route_cases as R
import test_gpu_conv_routes as T

pytestmark = pytest.mark.gpu

DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DIMS = (33, 18, 10)
# (BN, KC) -> (cin, cout): cout < BN leaves a partial N tile; cin < KC zero-fills the box's channels past the input's
CONFIGS = {(32, 64): (40, 24), (64, 32): (24, 40)}


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


@pytest.mark.parametrize("bn,kc,mode", [(bn, kc, m) for (bn, kc) in CONFIGS for m in (0, 1)], ids=lambda v: str(v))
def test_pair_matches_fp64(L, bn, kc, mode):
    cin, cout = CONFIGS[(bn, kc)]
    case = R.ConvCase("pair", bn, kc, False, mode, 1, "k3s1", cin, cout, DIMS)
    gen = torch.Generator().manual_seed(zlib.crc32(("pair-%d-%d-%d" % (bn, kc, mode)).encode()))
    if mode == 0:
        T.run_mode0(L, case, gen)
        T.run_mode0(L, case, gen, ext=L.diag_ext(max_ctas=5))
    else:
        for slope in (0.0, 0.01):
            T.run_mode1(L, case, gen, slope)


# ---------------------------------------------------------------------------------------------- C2 shapes, bit for bit
C2 = {"fwd": (64, 32, ("pair", 32, 64)), "dgrad": (32, 64, ("pair", 64, 32))}


def run_c2(L, which):
    """the C2 launch `which` on seeded device inputs: (route, stored output as int16, statistics)"""
    cin, cout, _ = C2[which]
    n, r = 2, 128
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(which.encode()))
    x = L.Act.empty(n, r, r, r, cin)
    x.hi.normal_(generator=g)
    w = torch.randn(cout, cin, 3, 3, 3, device=DEV, generator=g) / (cin * 27) ** 0.5
    whi, wlo, cop, cip, _ = L.pack_weights(w, 0)
    y = L.Act.empty(n, r, r, r, cout)
    y.hi.fill_(T.SENTINEL)
    st = torch.zeros(n, cout, 2, dtype=torch.float64, device=DEV)
    if which == "fwd":
        kw = dict(stats=st, stats_ld=cout)
    else:
        gx = L.Act.empty(n, r, r, r, cout)
        gx.hi.normal_(generator=g)
        coef = torch.rand(n, cout, 4, device=DEV, generator=g) - 0.5
        kw = dict(mode=1, gn_x=gx, coef=coef, coef_ld=cout, slope=0.01, bstats=st)
    route = L.conv3d_route(x, whi, wlo, 3, 1, y, cop, cip, **kw)
    L.conv3d(x, whi, wlo, 3, 1, y, cop, cip, **kw)
    torch.cuda.synchronize()
    return (route["kind"], route["bn"], route["kc"]), y.hi.view(torch.int16).cpu(), st.cpu()


def _child(which, path):
    import importlib
    L = importlib.import_module("3dunetcnn_b200").lib
    L.load_library()
    torch.save(run_c2(L, which), path)


@pytest.mark.parametrize("which", list(C2))
def test_c2_shape_is_bit_identical_to_per_tap_tiles(L, which, tmp_path):
    route, y, st = run_c2(L, which)
    assert route == C2[which][2]
    path = str(tmp_path / "tap.pt")
    env = dict(os.environ, B200UNET_NO_HALO="1")
    code = "import sys; sys.path[:0] = [%r, %r]; import %s as M; M._child(%r, %r)" % (ROOT, HERE, __name__.split(".")[-1], which, path)
    subprocess.run([sys.executable, "-c", code], env=env, check=True, cwd=ROOT)
    route_t, y_t, st_t = torch.load(path)
    assert route_t == ("tap",) + C2[which][2][1:]
    assert torch.equal(y, y_t), "%d of %d output elements differ" % (int((y != y_t).sum()), y.numel())
    assert bool(((st - st_t).abs() <= 1e-5 * st_t.abs().amax()).all()), "statistics differ beyond fp32 partial-sum rounding"
