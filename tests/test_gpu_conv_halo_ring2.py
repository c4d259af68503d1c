"""The (BN 64, KC 64) halo convolutions on the weight-only ring, two CTAs per SM (k_igemm_conv, ConvCfg::W_RING).

- Against fp64 at the bounds of tests/test_gpu_conv_routes.py, on the odd-extent halo plane (partial h and w tiles): the forward
  with residual, dropout scale and statistics, the mode-1 data gradient, fused 1x1x1 sources of 8, 32 and 96 channels (one and
  two K chunks, read after the taps from the drained halo box), and 48 output channels (a partial N tile).
- Bit for bit against the same launch on per-tap tiles (B200UNET_NO_HALO=1, in a child process): with one K chunk of the 3x3x3
  source both accumulate every output row in the same order (taps 0..26, then the fused source's chunks).  The per-channel
  statistics sum other fp32 per-tile partials, so they agree to fp32 rounding only.  Two launches of the same case store the
  same bits."""
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


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


# -------------------------------------------------------------------------------------------------------------- vs fp64
_C = R.ConvCase
FP64_CASES = [
    _C("halo", 64, 64, False, 0, 1, "k3s1", 64, 64, R.H),
    _C("halo", 64, 64, False, 1, 1, "k3s1", 64, 64, R.H),
    _C("halo", 64, 64, False, 0, 2, "k3s1", 64, 64, R.H, cin2=8, kchunks=(1, 1)),
    _C("halo", 64, 64, False, 0, 2, "k3s1", 64, 64, R.H, cin2=32, kchunks=(1, 1)),
    _C("halo", 64, 64, False, 0, 2, "k3s1", 64, 64, R.H, cin2=96, kchunks=(1, 2)),
    _C("halo", 64, 64, False, 1, 2, "k3s1", 64, 64, R.H, cin2=96, kchunks=(1, 2)),
    _C("halo", 64, 64, False, 0, 1, "k3s1", 48, 48, R.H),
    _C("halo", 64, 64, False, 1, 1, "k3s1", 48, 48, R.H),
]


def fp64_id(c):
    return "m%d-cin%d-cout%d-x%d" % (c.mode, c.cin, c.cout, c.cin2)


@pytest.mark.parametrize("case", FP64_CASES, ids=fp64_id)
def test_ring2_matches_fp64(L, case):
    gen = torch.Generator().manual_seed(zlib.crc32(("ring2-" + fp64_id(case)).encode()))
    if case.mode == 0:
        T.run_mode0(L, case, gen)
    else:
        for slope in (0.0, 0.01):
            T.run_mode1(L, case, gen, slope)


# -------------------------------------------------------------------------------------------------- vs per-tap, bit for bit
# name -> (mode, cin, cout, cin2, (n, d, h, w), forward extras)
BIT_CASES = {
    "fwd-plain": (0, 64, 64, 0, (2, 16, 64, 64), ()),
    "fwd-res-scale-stats": (0, 64, 64, 0, (2, 9, 33, 20), ("res", "scale", "stats")),
    "dgrad-mode1": (1, 64, 64, 0, (2, 9, 33, 20), ()),
    "fwd-sample8": (0, 64, 64, 8, (1, 16, 48, 40), ("stats",)),
    "fwd-sample32": (0, 64, 64, 32, (2, 8, 32, 32), ("res", "stats")),
    "fwd-sample96": (0, 64, 48, 96, (1, 16, 48, 40), ("stats",)),
    "fwd-cout48": (0, 48, 48, 0, (1, 12, 20, 16), ("res", "scale", "stats")),
}


def run_bits(L, name):
    """the case `name` on seeded device inputs: (route key, stored output as int16, statistics)"""
    mode, cin, cout, cin2, (n, d, h, w), extras = BIT_CASES[name]
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(name.encode()))
    x = L.Act.empty(n, d, h, w, cin)
    x.hi.normal_(generator=g)
    wt = torch.randn(cout, cin, 3, 3, 3, device=DEV, generator=g) / (cin * 27) ** 0.5
    whi, wlo, cop, cip, _ = L.pack_weights(wt, 0)
    kw = {}
    if cin2:
        x2 = L.Act.empty(n, d, h, w, cin2)
        x2.hi.normal_(generator=g)
        w2 = torch.randn(cout, cin2, 1, 1, 1, device=DEV, generator=g) / cin2 ** 0.5
        w2hi, w2lo, _, cip2, _ = L.pack_weights(w2, 0)
        kw.update(x2=x2, w2_hi=w2hi, w2_lo=w2lo, cip2=cip2)
    y = L.Act.empty(n, d, h, w, cout)
    y.hi.fill_(T.SENTINEL)
    st = torch.zeros(n, cout, 2, dtype=torch.float64, device=DEV)
    if mode == 0:
        if "res" in extras:
            res = L.Act.empty(n, d, h, w, cout)
            res.hi.normal_(generator=g)
            kw.update(res=res)
        if "scale" in extras:
            kw.update(scale=torch.tensor([0.0, 0.8, 1.25], device=DEV)[torch.randint(0, 3, (n, cout), device=DEV, generator=g)])
        if "stats" in extras:
            kw.update(stats=st, stats_ld=cout)
    else:
        gx = L.Act.empty(n, d, h, w, cout)
        gx.hi.normal_(generator=g)
        coef = torch.rand(n, cout, 4, device=DEV, generator=g) - 0.5
        kw.update(mode=1, gn_x=gx, coef=coef, coef_ld=cout, slope=0.01, bstats=st)
    route = L.conv3d_route(x, whi, wlo, 3, 1, y, cop, cip, **kw)
    L.conv3d(x, whi, wlo, 3, 1, y, cop, cip, **kw)
    torch.cuda.synchronize()
    out = (y.hi.view(torch.int16).cpu(), st.cpu())
    y.hi.fill_(T.SENTINEL)
    L.conv3d(x, whi, wlo, 3, 1, y, cop, cip, **kw)
    torch.cuda.synchronize()
    assert torch.equal(out[0], y.hi.view(torch.int16).cpu()), "a second launch stored other bits"
    key = (route["kind"], route["bn"], route["kc"], route["kchunks"], route["blocks_per_sm"])
    return key, out[0], out[1]


def _child(name, path):
    import importlib
    L = importlib.import_module("3dunetcnn_b200").lib
    L.load_library()
    torch.save(run_bits(L, name), path)


@pytest.mark.parametrize("name", list(BIT_CASES))
def test_ring2_is_bit_identical_to_per_tap_tiles(L, name, tmp_path):
    key, y, st = run_bits(L, name)
    cin2 = BIT_CASES[name][3]
    kchunks = (1, -(-cin2 // 64))
    assert key == ("halo", 64, 64, kchunks, 2), key
    path = str(tmp_path / "tap.pt")
    env = dict(os.environ, B200UNET_NO_HALO="1")
    code = "import sys; sys.path[:0] = [%r, %r]; import %s as M; M._child(%r, %r)" % (ROOT, HERE, __name__.split(".")[-1], name, path)
    subprocess.run([sys.executable, "-c", code], env=env, check=True, cwd=ROOT)
    key_t, y_t, st_t = torch.load(path)
    assert key_t[:4] == ("tap", 64, 64, kchunks), key_t
    assert torch.equal(y, y_t), "%d of %d output elements differ" % (int((y != y_t).sum()), y.numel())
    assert bool(((st - st_t).abs() <= 1e-5 * st_t.abs().amax()).all()), "statistics differ beyond fp32 partial-sum rounding"
