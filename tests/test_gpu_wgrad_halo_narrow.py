"""The halo weight gradient at the C2 channel widths (one 64-channel box per voxel tile, zero-filled past 8..32 input channels,
two consumer warpgroups per CTA) against fp64, on an output plane that fills the 8 x 16 halo tile with partial tiles in h and w:
atomic and deterministic accumulation, the network's first layer with 4 real channels in an 8-channel view, and a dY whose
visible extents are one short.  32 -> 64 stays on per-tap tiles (N tile 64) and is checked the same way."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"
DIMS = (2, 18, 12)      # 3 x 2 x 2 halo tiles of 8 x 16 x 1 per sample, the last in h and w partial
PAIRS = [(8, 32, 4), (16, 16, 16), (32, 32, 32), (64, 32, 64), (32, 64, 32)]   # (ci, co, real input channels)


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


def rel(a, b):
    return float((a.double().cpu() - b).norm() / b.norm())


def inputs(L, ci, co, real, seed, dy_vis=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.zeros(2, ci, *DIMS)
    x[:, :real] = torch.randn(2, real, *DIMS, generator=g)
    a = L.Act.from_ncdhw(x.to(DEV))
    dy = L.Act.from_ncdhw(torch.randn(2, co, *DIMS, generator=g).to(DEV))
    dyv = dy.to_ncdhw(co).double().cpu()
    if dy_vis:   # the kernel reads dY only inside its visible extents
        dyv[:, :, dy_vis[0]:] = 0
        dyv[:, :, :, dy_vis[1]:] = 0
        dyv[..., dy_vis[2]:] = 0
    wz = torch.zeros(co, ci, 3, 3, 3, dtype=torch.float64, requires_grad=True)
    F.conv3d(a.to_ncdhw(ci).double().cpu(), wz, padding=1).backward(dyv)
    ref = wz.grad.permute(2, 3, 4, 1, 0).reshape(27, ci, co)     # dw[tap][ci][co]
    return a, dy, ref


def check_route(L, a, dy, ci, co, **kw):
    r = L.wgrad_route(a, dy, 3, 1, ci, co, num_sms=torch.cuda.get_device_properties(0).multi_processor_count, **kw)
    halo = ci > 32 or co <= 32
    assert (r["kind"], r["cb"]) == (("halo", 64) if halo else ("tap", 32 if ci > 16 else 16)), r
    return r


@pytest.mark.parametrize("ci,co,real", PAIRS)
def test_halo_wgrad_matches_fp64(L, ci, co, real):
    a, dy, ref = inputs(L, ci, co, real, ci * 100 + co)
    check_route(L, a, dy, ci, co)
    dw = torch.zeros(27, ci, co, device=DEV)
    assert L.wgrad_ex(a, dy, 3, 1, ci, co, dw) == 0
    torch.cuda.synchronize()
    assert rel(dw, ref) < 1e-5
    if real < ci:   # the padded input channels of the first layer: their gradient rows stay exactly zero
        assert torch.count_nonzero(dw[:, real:]) == 0


@pytest.mark.parametrize("ci,co,real", PAIRS)
def test_halo_wgrad_deterministic(L, ci, co, real):
    a, dy, ref = inputs(L, ci, co, real, ci * 100 + co + 1)
    rd = check_route(L, a, dy, ci, co, deterministic=True)
    part = torch.empty(L.wgrad_partial_bytes(a, dy, 3, 1, ci, co) // 4, device=DEV)
    outs = []
    for _ in range(2):
        dw = torch.full((27, ci, co), float("nan"), device=DEV)
        assert L.wgrad_ex(a, dy, 3, 1, ci, co, dw, part=part) == rd["splits"]
        torch.cuda.synchronize()
        outs.append(dw)
    assert torch.equal(outs[0], outs[1]), "deterministic weight gradient differs between two runs"
    assert rel(outs[0], ref) < 1e-5
    dwa = torch.zeros(27, ci, co, device=DEV)
    L.wgrad_ex(a, dy, 3, 1, ci, co, dwa)
    torch.cuda.synchronize()
    # the same fp32 products summed in another order
    assert float((dwa - outs[0]).norm() / outs[0].norm()) < 1e-6


@pytest.mark.parametrize("ci,co,real", [(8, 32, 4), (32, 32, 32)])
def test_halo_wgrad_dy_visible_extents_one_short(L, ci, co, real):
    vis = tuple(v - 1 for v in DIMS)
    a, dy, ref = inputs(L, ci, co, real, 7, dy_vis=vis)
    ext = L.diag_ext(dy_vis=vis)
    check_route(L, a, dy, ci, co, ext=ext)
    dw = torch.zeros(27, ci, co, device=DEV)
    L.wgrad_ex(a, dy, 3, 1, ci, co, dw, ext=ext)
    torch.cuda.synchronize()
    assert rel(dw, ref) < 1e-5
