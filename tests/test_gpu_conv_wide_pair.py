"""The 256-voxel per-tap tile (k_igemm_conv_wide): BN = 128, two consumer warpgroups sharing each weight tile.

Each shape class (3x3x3 stride 1, stride 2, 1x1x1, a fused 1x1x1 second source), in both epilogue modes and both precisions,
on 2 x 12 x 18 x 30 output voxels and 200 output channels: 160 CTAs of 256 voxels, partial on every axis and in N, and the
second warpgroup of the last depth tile wholly outside the volume.  The K chunks cover KC 16, 32 and 64.

- Against fp64 at the bounds of tests/test_gpu_conv_routes.py.
- Bit for bit against the same launch on the 128-voxel tile (the diagnostics option tile128): every output row sees the same
  MMA order.  The statistics sum the same per-warpgroup fp32 partials, in another order of the fp64 atomics."""
import zlib

import pytest
import torch

import conv_route_cases as R
import test_gpu_conv_routes as T

pytestmark = pytest.mark.gpu

DEV = "cuda"
DIMS = (12, 18, 30)
_C = R.ConvCase
CASES = [
    _C("tap", 128, 64, False, 0, 1, "k3s1", 72, 200, DIMS, kchunks=(2, 0)),
    _C("tap", 128, 16, False, 0, 1, "k3s2", 16, 200, DIMS),
    _C("tap", 128, 64, False, 0, 1, "k1", 136, 200, DIMS, kchunks=(3, 0)),
    _C("tap", 128, 64, False, 0, 2, "k3s1", 72, 200, DIMS, cin2=40, kchunks=(2, 1)),
    _C("tap", 128, 32, False, 0, 2, "k3s2", 24, 200, DIMS, cin2=40, kchunks=(1, 2)),
]
CASES = [_C(c.kind, c.bn, c.kc, split, mode, c.nsrc, c.op, c.cin, c.cout, c.dims, c.cin2, c.kchunks)
         for c in CASES for split in (False, True) for mode in (0, 1)]


def case_id(c):
    return "%s-%s%s" % (c.id, c.op, "+%d" % c.cin2 if c.cin2 else "")


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


def wide_route(L, args, kw, ext=None):
    x, whi, wlo, ksz, stride, out, cop, cip = args
    return L.conv3d_route(x, whi, wlo, ksz, stride, out, cop, cip, ext=ext, **kw)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_wide_tile_matches_fp64(L, case):
    gen = torch.Generator().manual_seed(zlib.crc32(case_id(case).encode()))
    if case.mode == 0:
        r = T.run_mode0(L, case, gen)
        assert r["wgs"] == 2 and (r["tw"], r["th"], r["td"]) == (8, 4, 8), r
    else:
        for slope in (0.0, 0.01):
            T.run_mode1(L, case, gen, slope)


def test_wide_tile_bias_and_zeroed_boundary(L):
    """the transposed-convolution epilogue of the plans (tests/test_gpu_conv_routes.py: test_conv_bias_and_zeroed_boundary)"""
    case = CASES[0]
    gen = torch.Generator().manual_seed(13)
    bias = torch.zeros(case.cout)
    bias[:case.cout - 4] = torch.randn(case.cout - 4, generator=gen)
    bias = bias.to(DEV)

    def edit(ref, bound):
        ref = ref + bias.double().cpu()[None, :case.cout - 4, None, None, None]
        for t in (ref, bound):
            t[:, :, -1] = 0
            t[:, :, :, -1] = 0
            t[..., -1] = 0
        return ref, bound
    r = T.run_mode0(L, case, gen, ext=L.diag_ext(bias=bias, zero_last=True), edit_ref=edit)
    assert r["wgs"] == 2


def run_both(L, case):
    """the case on seeded device inputs with the 256- and with the 128-voxel tile: [(route, hi, lo, stats)] per tile"""
    n = 2
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(("bits-" + case_id(case)).encode()))
    sdims, ksz, stride, _ = R.conv_geometry(case.op, case.cin, case.dims)

    def act(dims, c):
        a = L.Act.empty(n, *dims, c, split=case.split)
        a.hi.normal_(generator=g)
        if case.split:
            a.lo.copy_((torch.randn(a.lo.shape, device=DEV, generator=g) * 2.0 ** -9).bfloat16())
        return a

    def weights(ci, k):
        w = torch.randn(case.cout, ci, k, k, k, device=DEV, generator=g) / (ci * k ** 3) ** 0.5
        return L.pack_weights(w, 0, split=case.split)

    x = act(sdims, case.cin)
    whi, wlo, cop, cip, _ = weights(case.cin, ksz)
    kw = {}
    if case.cin2:
        w2hi, w2lo, _, cip2, _ = weights(case.cin2, 1)
        kw.update(x2=act(case.dims, case.cin2), w2_hi=w2hi, w2_lo=w2lo, cip2=cip2)
    st = torch.zeros(n, case.cout, 2, dtype=torch.float64, device=DEV)
    if case.mode == 0:
        kw.update(res=act(case.dims, case.cout), scale=torch.rand(n, case.cout, device=DEV, generator=g) + 0.5, stats=st,
                  stats_ld=case.cout)
    else:
        kw.update(mode=1, gn_x=act(case.dims, case.cout), coef=torch.rand(n, case.cout, 4, device=DEV, generator=g) - 0.5,
                  coef_ld=case.cout, slope=0.01, bstats=st)
    got = []
    for tile128 in (False, True):
        y = L.Act.empty(n, *case.dims, case.cout, split=case.split)
        y.hi.fill_(float("nan"))
        if case.split:
            y.lo.fill_(float("nan"))
        st.zero_()
        ext = L.diag_ext(tile128=tile128)
        args = (x, whi, wlo, ksz, stride, y, cop, cip)
        route = wide_route(L, args, kw, ext)
        L.conv3d_ex(*args, ext=ext, **kw)
        torch.cuda.synchronize()
        got.append((route, y.hi.view(torch.int16).cpu(), y.lo.view(torch.int16).cpu() if case.split else None, st.cpu()))
    return got


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_wide_tile_is_bit_identical_to_the_128_voxel_tile(L, case):
    (r, hi, lo, st), (r1, hi1, lo1, st1) = run_both(L, case)
    T.assert_route(r, case)
    T.assert_route(r1, case)
    assert (r["wgs"], r["td"], r1["wgs"], r1["td"]) == (2, 8, 1, 4), (r, r1)
    assert not bool(hi1.view(torch.bfloat16).isnan().any()), "the 128-voxel tile left an output unwritten"
    assert torch.equal(hi, hi1), "%d of %d output elements differ" % (int((hi != hi1).sum()), hi.numel())
    if case.split:
        assert torch.equal(lo, lo1), "%d of %d lo elements differ" % (int((lo != lo1).sum()), lo.numel())
    assert bool(((st - st1).abs() <= 1e-5 * st1.abs().amax()).all()), "statistics differ beyond fp32 partial-sum rounding"
