"""The persistent, weight-stationary halo kernel with several voxel tiles per CTA.

At the sizes of tests/test_gpu_conv_routes.py every CTA gets one tile.  Here the diagnostics cap `max_ctas` makes one or three
CTAs walk all 24 tiles of a (3, 18, 10) output, batch 2, for every (BN, KC) the kernel serves, in both epilogue modes, with one
source and with a fused 1x1x1 second source of two K chunks, and with a partial last N tile.  The stored output must not depend
on the cap (same bits: each output row accumulates in the same order whichever CTA computes it), the per-channel statistics may
differ only by the order of their fp64 atomics, and the result must match fp64 within the bounds of the route tests."""
import zlib

import pytest
import torch
import torch.nn.functional as F

import conv_route_cases as R
import test_gpu_conv_routes as T

pytestmark = pytest.mark.gpu

DEV = "cuda"
DIMS = (3, 18, 10)        # 3 x 2 x 2 halo tiles per sample, partial along H and W
CAPS = (1, 3, 0)          # 0: the default grid (one CTA per tile at this size)
# (BN, KC) -> (cin, cout, cin2 of two K chunks): cout = BN - 8 leaves a partial N tile, BN 16 with cout 8 too
CONFIGS = {(16, 16): (16, 8, 32), (16, 32): (24, 8, 40), (32, 16): (16, 24, 24), (32, 32): (24, 24, 64),
           (64, 16): (8, 40, 32), (64, 32): (32, 40, 48)}
PARAMS = [(bn, kc, mode, nsrc) for (bn, kc) in CONFIGS for mode in (0, 1) for nsrc in (1, 2)]


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


def stats_close(a, b):
    """fp64 sums of the same fp32 per-tile partials, added in another order (an fp32 sum across tiles would be ~1e-7 off)"""
    return bool(((a - b).abs() <= 1e-10 * a.abs().amax() + 1e-30).all())


@pytest.mark.parametrize("bn,kc,mode,nsrc", PARAMS, ids=lambda v: str(v))
def test_several_tiles_per_cta(L, bn, kc, mode, nsrc):
    cin, cout, cin2 = CONFIGS[(bn, kc)]
    cin2 = cin2 if nsrc == 2 else 0
    case = R.ConvCase("halo", bn, kc, False, mode, nsrc, "k3s1", cin, cout, DIMS, cin2=cin2,
                      kchunks=(1, 2 if nsrc == 2 else 0))
    gen = torch.Generator().manual_seed(zlib.crc32(("persistent-%d-%d-%d-%d" % (bn, kc, mode, nsrc)).encode()))
    n = 2
    args, kw, acc, absacc = T.conv_inputs(L, case, gen, cout)
    x, whi, wlo, ksz, stride = args
    side, sidev = T.rand_act(L, n, cout, DIMS, False, gen, shift=0.3 if mode == 1 else 0.0)
    if mode == 0:
        scale = torch.tensor([0.0, 0.8, 1.25])[torch.randint(0, 3, (n, cout), generator=gen)].to(DEV)
        kw.update(res=side, scale=scale, stats_ld=cout)
    else:
        gamma = (torch.randn(cout, generator=gen) * 0.3 + 1).to(DEV)
        beta = (torch.randn(cout, generator=gen) * 0.2).to(DEV)
        st_in = torch.stack([sidev.sum(dim=(2, 3, 4)), (sidev * sidev).sum(dim=(2, 3, 4))], dim=-1).contiguous().to(DEV)
        coef = torch.empty(n, cout, 4, device=DEV)
        L.gn_apply(side, L.Act.empty(n, *DIMS, cout), st_in, gamma, beta, cout, T.G, coef, slope=0.01)
        kw.update(mode=1, gn_x=side, coef=coef, coef_ld=cout, slope=0.01)

    tiles = 2 * 3 * 2 * 2
    outs, stats = [], []
    for cap in CAPS:
        st = torch.zeros(n, cout, 2, dtype=torch.float64, device=DEV)
        kw.update(stats=st) if mode == 0 else kw.update(bstats=st)
        y = L.Act.empty(n, *DIMS, cout)
        y.hi.fill_(T.SENTINEL)
        ext = L.diag_ext(max_ctas=cap)
        r = L.conv3d_route(x, whi, wlo, ksz, stride, y, cout, cin, ext=ext, **kw)
        T.assert_route(r, case)
        assert r["grid"] == ((cap or tiles), 1, 1), r
        L.conv3d_ex(x, whi, wlo, ksz, stride, y, cout, cin, ext=ext, **kw)
        torch.cuda.synchronize()
        outs.append(y.hi.clone())
        stats.append(st.cpu())
    for cap, o, s in zip(CAPS[:-1], outs[:-1], stats[:-1]):
        assert torch.equal(o.view(torch.int16), outs[-1].view(torch.int16)), "output differs with max_ctas=%d" % cap
        assert stats_close(s, stats[-1]), "statistics differ with max_ctas=%d beyond fp64 rounding" % cap

    # against fp64, as tests/test_gpu_conv_routes.py bounds it
    got = T.view_value(y)
    bound = T.A_ACC * absacc
    dims = (2, 3, 4)
    st = stats[-1]
    if mode == 0:
        s = scale.double().cpu()[:, :, None, None, None]
        ref = (acc + sidev) * s
        bound = bound * s
        T.check_elements(got, ref, bound, T.R_STORE[False], "output")
        b1 = bound.sum(dim=dims) + 2.0 ** -16 * ref.abs().sum(dim=dims) + 1e-9
        b2 = (2 * ref.abs() * bound + bound * bound).sum(dim=dims) + 2.0 ** -16 * (ref * ref).sum(dim=dims) + 1e-9
        assert bool(((st[..., 0] - ref.sum(dim=dims)).abs() <= b1).all()), "per-channel sums"
        assert bool(((st[..., 1] - (ref * ref).sum(dim=dims)).abs() <= b2).all()), "per-channel sums of squares"
    else:
        xq = sidev.clone().requires_grad_(True)
        z = F.group_norm(xq, T.G, gamma.double().cpu(), beta.double().cpu(), 1e-5)
        z.retain_grad()
        F.leaky_relu(z, 0.01).backward(acc)
        ref = z.grad
        clear = z.detach().abs() > 1e-3
        T.check_elements(got, ref, bound, T.R_STORE[False], "dz", mask=clear)
        mu, rstd = coef[..., 2].double().cpu(), coef[..., 3].double().cpu()
        xhat = (sidev - mu[:, :, None, None, None]) * rstd[:, :, None, None, None]
        amb = (~clear).double() * acc.abs()
        b1 = bound.sum(dim=dims) + amb.sum(dim=dims) + 2.0 ** -16 * ref.abs().sum(dim=dims) + 1e-9
        b2 = ((bound + amb) * xhat.abs()).sum(dim=dims) + 2.0 ** -16 * (ref * xhat).abs().sum(dim=dims) + 1e-9
        assert bool(((st[..., 0] - ref.sum(dim=dims)).abs() <= b1).all()), "sum dz"
        assert bool(((st[..., 1] - (ref * xhat).sum(dim=dims)).abs() <= b2).all()), "sum dz * xhat"


def test_grid_is_one_wave_at_full_size(L):
    """at 2 x 128^3 the grid holds blocks_per_sm x SMs CTAs, far fewer than the 2 x 128 x 8 x 16 tiles"""
    r = R.conv_query(L, "k3s1", 32, 32, (128, 128, 128))
    assert (r["kind"], r["bn"], r["kc"], r["blocks_per_sm"]) == ("halo", 32, 32, 2)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert r["grid"] == (2 * sms, 1, 1)
