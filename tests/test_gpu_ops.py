"""Per-kernel parity on the GPU, through the C ABI, against the CPU oracle (torch CPU fp64 ops / numpy restatements)
on the same seeded inputs.  Tolerances: the kernels take bf16 operands (single pass) or hi/lo bf16 pairs (split);
inputs are quantised to exactly what the kernel reads before the oracle sees them, so the remaining error is fp32
accumulation + the bf16 (2^-9) or hi/lo (2^-17) rounding of the stored result."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import conv3d_direct, dice_loss, group_norm, trilinear_upsample2x

pytestmark = pytest.mark.gpu

TOL_STORE = {False: 4e-3, True: 5e-5}      # rel-L2 of a stored activation: bf16 / hi+lo
DEV = "cuda"


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _channel_stats(a):
    """fp64 (sum, sumsq) [n][a.c][2] of every channel of view a, from the stored values: what the epilogue of the producing
    convolution accumulates for the next GroupNorm"""
    v = a.value().double()
    return torch.stack([v.sum(dim=(1, 2, 3)), (v * v).sum(dim=(1, 2, 3))], dim=-1).contiguous()


def _packed_to_torch(L, w, mode, split, cout, cin, ksz):
    hi, lo, cop, cip, T = L.pack_weights(w, mode, split=split)
    q = hi.float() + (lo.float() if split else 0)
    return hi, lo, cop, cip, q.double().cpu()[:, :cout, :cin].reshape(ksz, ksz, ksz, cout, cin).permute(3, 4, 0, 1, 2)


# the forward shapes below that run on the halo kernel in bf16; (64, 32) has KC = 64 with BN = 32 and stays on per-tap tiles
# (halo_keeps_occupancy), inputs wider than 64 channels unless B200UNET_HALO_WIDE_MIN allows them
HALO_FORWARD = {(32, 32, (8, 16, 16)), (8, 32, (16, 16, 16)), (24, 40, (6, 18, 12)), (32, 64, (5, 24, 20)), (16, 16, (1, 16, 8))}


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("cin,cout,dims,ksz,stride", [
    (64, 64, (8, 8, 8), 3, 1), (32, 32, (8, 8, 16), 3, 1), (8, 32, (8, 8, 8), 3, 1), (128, 128, (4, 8, 8), 3, 1),
    (256, 256, (4, 4, 8), 3, 1), (24, 40, (5, 7, 9), 3, 1), (96, 192, (4, 4, 8), 3, 1), (64, 32, (8, 8, 8), 3, 1),
    (256, 128, (4, 4, 8), 1, 1), (8, 32, (6, 6, 6), 1, 1), (32, 32, (16, 16, 16), 3, 2), (64, 64, (8, 8, 8), 3, 2),
    (16, 16, (10, 6, 14), 3, 2),
    # output plane >= 8 x 16: the halo kernel in bf16 where HALO_FORWARD lists it (the route is asserted)
    (32, 32, (8, 16, 16), 3, 1), (64, 32, (4, 16, 8), 3, 1), (8, 32, (16, 16, 16), 3, 1), (128, 128, (8, 16, 8), 3, 1),
    (256, 256, (2, 16, 8), 3, 1), (24, 40, (6, 18, 12), 3, 1), (96, 192, (3, 16, 8), 3, 1), (32, 64, (5, 24, 20), 3, 1),
    (16, 16, (1, 16, 8), 3, 1),
    # 1x1x1 with a large output plane (per-tap tiles)
    (32, 64, (4, 16, 8), 1, 1), (8, 32, (5, 18, 12), 1, 1), (64, 32, (2, 16, 16), 1, 1), (24, 40, (3, 16, 9), 1, 1),
])
def test_conv3d_forward(pkg, cin, cout, dims, ksz, stride, split):
    L = pkg.lib
    torch.manual_seed(cin * 7 + cout)
    n = 2
    x = torch.randn(n, cin, *dims, device=DEV)
    w = torch.randn(cout, cin, ksz, ksz, ksz, device=DEV) / (cin * ksz ** 3) ** 0.5
    a = L.Act.from_ncdhw(x, split=split)
    whi, wlo, cop, cip, wq = _packed_to_torch(L, w, 0, split, cout, cin, ksz)
    pad = ksz // 2
    od = [(s + 2 * pad - ksz) // stride + 1 for s in dims]
    y = L.Act.empty(n, *od, cop, split=split, zero=True)
    halo = not split and (cin, cout, dims) in HALO_FORWARD
    assert L.conv3d_route(a, whi, wlo, ksz, stride, y, cop, cip)["kind"] == ("halo" if halo else "tap")
    L.conv3d(a, whi, wlo, ksz, stride, y, cop, cip)
    ref = F.conv3d(a.to_ncdhw(cin).double().cpu(), wq, stride=stride, padding=pad)
    assert rel(y.to_ncdhw(cout), ref) < TOL_STORE[split]
    if cop > cout:                                            # padded output channels stay zero
        assert float(y.hi[..., cout:].float().abs().max()) == 0.0


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("cin,cout,dims,mode", [
    (128, 128, (4, 16, 8), "plain"), (256, 192, (2, 16, 16), "plain"), (96, 160, (6, 16, 8), "plain"),
    (128, 128, (5, 16, 16), "res"), (256, 256, (3, 16, 8), "res"),
])
def test_conv3d_wide_inputs_on_halo_kernel(pkg, monkeypatch, cin, cout, dims, mode, split):
    """Cin >= 128 in halo mode (bf16; several N tiles per voxel tile, 2-4 halo boxes per tile).  That dispatch is off by
    default and enabled here through B200UNET_HALO_WIDE_MIN so that it stays correct.  Split precision runs on per-tap
    tiles."""
    monkeypatch.setenv("B200UNET_HALO_WIDE_MIN", "0")
    L = pkg.lib
    torch.manual_seed(cin * 3 + cout)
    n = 2
    x = torch.randn(n, cin, *dims, device=DEV)
    w = torch.randn(cout, cin, 3, 3, 3, device=DEV) / (cin * 27) ** 0.5
    a = L.Act.from_ncdhw(x, split=split)
    whi, wlo, cop, cip, wq = _packed_to_torch(L, w, 0, split, cout, cin, 3)
    y = L.Act.empty(n, *dims, cop, split=split, zero=True)
    stats = torch.zeros(n, cop, 2, dtype=torch.float64, device=DEV)
    ref = F.conv3d(a.to_ncdhw(cin).double().cpu(), wq, padding=1)
    assert L.conv3d_route(a, whi, wlo, 3, 1, y, cop, cip)["kind"] == ("tap" if split else "halo")
    if mode == "res":
        assert cop == cout                                   # the shapes above need no channel padding
        r = L.Act.from_ncdhw(torch.randn(n, cout, *dims, device=DEV), split=split)
        L.conv3d(a, whi, wlo, 3, 1, y, cop, cip, res=r, stats=stats, stats_ld=cop)
        ref = ref + r.to_ncdhw(cout).double().cpu()
    else:
        L.conv3d(a, whi, wlo, 3, 1, y, cop, cip, stats=stats, stats_ld=cop)
    assert rel(y.to_ncdhw(cout), ref) < TOL_STORE[split]
    s_ref = torch.stack([ref.sum(dim=(2, 3, 4)), (ref * ref).sum(dim=(2, 3, 4))], dim=-1)
    assert rel(stats[:, :cout].cpu(), s_ref) < (2e-3 if not split else 1e-4)


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("ci,co,dims", [(128, 128, (4, 16, 8)), (192, 256, (2, 16, 16)), (128, 96, (5, 16, 8))])
def test_conv3d_wide_inputs_on_halo_kernel_gn_backward_epilogue_on_fused_coefficients(pkg, monkeypatch, ci, co, dims, split):
    """The same wide-input halo-mode dispatch with the mode-1 (GroupNorm/ReLU backward) epilogue: the data gradient of a
    co -> ci ... convolution seen from its output side, i.e. K = co >= 128 input channels of the GEMM."""
    monkeypatch.setenv("B200UNET_HALO_WIDE_MIN", "0")
    L = pkg.lib
    torch.manual_seed(ci + 2 * co)
    n, G = 2, 8
    dyv = torch.randn(n, co, *dims, device=DEV)
    xv = torch.randn(n, ci, *dims, device=DEV) + 0.3
    w = torch.randn(co, ci, 3, 3, 3, device=DEV) / (ci * 27) ** 0.5
    gamma, beta = torch.randn(ci, device=DEV) * 0.3 + 1, torch.randn(ci, device=DEV) * 0.2
    dy, x = L.Act.from_ncdhw(dyv, split=split), L.Act.from_ncdhw(xv, split=split)
    wdh, wdl, _, _, _ = L.pack_weights(w, 1, split=split)
    _, _, _, _, wq = _packed_to_torch(L, w, 0, split, co, ci, 3)
    coef = torch.empty(n, ci, 4, device=DEV)
    L.gn_apply(x, L.Act.empty(n, *dims, ci, split=split), _channel_stats(x), gamma, beta, ci, G, coef)
    bst = torch.zeros(n, ci, 2, dtype=torch.float64, device=DEV)
    dz = L.Act.empty(n, *dims, ci, split=split)
    mode1 = dict(mode=1, gn_x=x, coef=coef, coef_ld=ci, bstats=bst)
    assert L.conv3d_route(dy, wdh, wdl, 3, 1, dz, ci, co, **mode1)["kind"] == ("tap" if split else "halo")
    L.conv3d(dy, wdh, wdl, 3, 1, dz, ci, co, **mode1)
    xq = x.to_ncdhw(ci).double().cpu().requires_grad_(True)
    z = F.group_norm(xq, G, gamma.double().cpu(), beta.double().cpu(), 1e-5)
    z.retain_grad()
    F.conv3d(F.relu(z), wq, padding=1).backward(dy.to_ncdhw(co).double().cpu())
    assert rel(dz.to_ncdhw(ci), z.grad) < TOL_STORE[split] * 1.5
    mu, rstd = coef[..., 2].double().cpu(), coef[..., 3].double().cpu()
    xhat = (xq.detach() - mu[:, :, None, None, None]) * rstd[:, :, None, None, None]
    b_ref = torch.stack([z.grad.sum(dim=(2, 3, 4)), (z.grad * xhat).sum(dim=(2, 3, 4))], dim=-1)
    assert rel(bst, b_ref) < (2e-3 if not split else 1e-4)


@pytest.mark.parametrize("cin,cout,r", [(32, 32, 64), (64, 64, 48), (64, 128, 32), (32, 64, 64), (128, 128, 32)])
def test_conv3d_outputs_are_bitwise_repeatable(pkg, cin, cout, r):
    """Race detector: the stored activations involve no atomics, so repeated launches on identical inputs must agree
    bit for bit (many persistent tiles per SM; a lost accumulate or a recycled staging buffer shows up here).
    Only the fp64 statistics may differ in the last bits (atomic order)."""
    L = pkg.lib
    torch.manual_seed(5)
    n = 2
    x = L.Act.empty(n, r, r, r, cin)
    x.hi.normal_()
    w = torch.randn(cout, cin, 3, 3, 3, device=DEV) / (cin * 27) ** 0.5
    whi, _, cop, cip, _ = L.pack_weights(w, 0)
    side = L.Act.empty(n, r, r, r, cout)
    side.hi.normal_()
    coef = torch.rand(n, cout, 4, device=DEV)
    for mode in ("plain", "res", "gn_bwd"):
        outs = []
        for _ in range(3):
            y = L.Act.empty(n, r, r, r, cout)
            y.hi.fill_(7.0)
            st = torch.zeros(n, cout, 2, dtype=torch.float64, device=DEV)
            if mode == "plain":
                L.conv3d(x, whi, None, 3, 1, y, cop, cip, stats=st, stats_ld=cout)
            elif mode == "res":
                L.conv3d(x, whi, None, 3, 1, y, cop, cip, res=side, stats=st, stats_ld=cout)
            else:
                L.conv3d(x, whi, None, 3, 1, y, cop, cip, mode=1, gn_x=side, coef=coef, coef_ld=cout, bstats=st)
            torch.cuda.synchronize()
            outs.append((y.hi.clone(), st.clone()))
        for o in outs[1:]:
            assert int((o[0] != outs[0][0]).sum()) == 0, mode
            assert float((o[1] - outs[0][1]).abs().max()) <= 1e-9 * float(outs[0][1].abs().max()), mode


def test_conv3d_vs_numpy_restatement(pkg):
    """tiny case against the plain-numpy cross-correlation (no torch arithmetic on the oracle side)."""
    L = pkg.lib
    rng = np.random.default_rng(0)
    x = torch.from_numpy(rng.standard_normal((1, 8, 4, 5, 6))).float().to(DEV)
    w = torch.from_numpy(rng.standard_normal((8, 8, 3, 3, 3)) * 0.1).float().to(DEV)
    a = L.Act.from_ncdhw(x, split=True)
    whi, wlo, cop, cip, wq = _packed_to_torch(L, w, 0, True, 8, 8, 3)
    y = L.Act.empty(1, 4, 5, 6, 8, split=True)
    L.conv3d(a, whi, wlo, 3, 1, y, cop, cip)
    ref = conv3d_direct(a.to_ncdhw(8).double().cpu().numpy(), wq.numpy(), 1, 1)
    assert rel(y.to_ncdhw(8), torch.from_numpy(ref)) < 5e-5


@pytest.mark.parametrize("split", [False, True])
def test_conv3d_fused_epilogue_residual_dropout_stats_concat_slice(pkg, split):
    """(acc + residual) * channel scale, written into the second half of a wider (concat) buffer, with the
    per-channel statistics the next GroupNorm consumes."""
    L = pkg.lib
    torch.manual_seed(1)
    n, ci, co, D = 2, 32, 32, 16
    x = torch.randn(n, ci, D, D, D, device=DEV)
    w = torch.randn(co, ci, 3, 3, 3, device=DEV) / (ci * 27) ** 0.5
    r = torch.randn(n, co, D, D, D, device=DEV)
    a, res = L.Act.from_ncdhw(x, split=split), L.Act.from_ncdhw(r, split=split)
    whi, wlo, cop, cip, wq = _packed_to_torch(L, w, 0, split, co, ci, 3)
    scale = ((torch.rand(n, co, device=DEV) > 0.3).float() * 1.25).contiguous()
    cat = L.Act.empty(n, D, D, D, 2 * co, split=split, zero=True)
    stats = torch.zeros(n, 2 * co, 2, dtype=torch.float64, device=DEV)
    epi = dict(res=res, scale=scale, stats=stats[:, co:], stats_ld=2 * co)
    assert L.conv3d_route(a, whi, wlo, 3, 1, cat.slice(co, co), cop, cip, **epi)["kind"] == ("tap" if split else "halo")
    L.conv3d(a, whi, wlo, 3, 1, cat.slice(co, co), cop, cip, **epi)
    ref = (F.conv3d(a.to_ncdhw(ci).double().cpu(), wq, padding=1) + res.to_ncdhw(co).double().cpu()) * scale.double().cpu()[:, :, None, None, None]
    got = cat.slice(co, co).to_ncdhw(co)
    assert rel(got, ref) < TOL_STORE[split]
    assert float(cat.hi[..., :co].float().abs().max()) == 0.0           # first half untouched
    gd = got.double()
    s_ref = torch.stack([gd.sum(dim=(2, 3, 4)), (gd * gd).sum(dim=(2, 3, 4))], dim=-1)
    assert rel(stats[:, co:], s_ref) < (2e-3 if not split else 1e-5)    # stats are taken before the bf16 rounding
    assert float(stats[:, :co].abs().max()) == 0.0


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("D", [8, 16])
def test_conv3d_two_sources_is_block_output(pkg, split, D):
    """conv2(a2) + sample(x): the residual block's second conv with the 1x1x1 `sample` as a second K-slab
    (D=8: per-tap tiles, D=16: the halo kernel in bf16)."""
    L = pkg.lib
    torch.manual_seed(2)
    n, ci, co = 1, 8, 32
    x = torch.randn(n, ci, D, D, D, device=DEV)
    h = torch.randn(n, co, D, D, D, device=DEV)
    w2 = torch.randn(co, co, 3, 3, 3, device=DEV) / (co * 27) ** 0.5
    ws = torch.randn(co, ci, 1, 1, 1, device=DEV) / ci ** 0.5
    ax, ah = L.Act.from_ncdhw(x, split=split), L.Act.from_ncdhw(h, split=split)
    w2h, w2l, cop, cip, w2q = _packed_to_torch(L, w2, 0, split, co, co, 3)
    wsh, wsl, _, cips, wsq = _packed_to_torch(L, ws, 0, split, co, ci, 1)
    y = L.Act.empty(n, D, D, D, co, split=split)
    route = L.conv3d_route(ah, w2h, w2l, 3, 1, y, cop, cip, x2=ax, w2_hi=wsh, w2_lo=wsl, cip2=cips)
    assert route["kind"] == ("halo" if D == 16 and not split else "tap")
    L.conv3d(ah, w2h, w2l, 3, 1, y, cop, cip, x2=ax, w2_hi=wsh, w2_lo=wsl, cip2=cips)
    ref = F.conv3d(ah.to_ncdhw(co).double().cpu(), w2q, padding=1) + F.conv3d(ax.to_ncdhw(ci).double().cpu(), wsq)
    assert rel(y.to_ncdhw(co), ref) < TOL_STORE[split]


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("D", [8, 16])
def test_conv3d_dgrad_groupnorm_relu_backward_epilogue_on_fused_coefficients(pkg, split, D):
    """dz = dgrad(dy) masked by ReLU'(GN(x)), plus per-channel (sum dz, sum dz*xhat): checked against autograd.  With K = 64 and
    32 outputs both extents run on per-tap tiles (halo_keeps_occupancy); the mode-1 epilogue on the halo kernel is covered by the
    halo mode-1 cases of tests/test_gpu_conv_routes.py."""
    L = pkg.lib
    torch.manual_seed(3)
    n, ci, co, G = 2, 32, 64, 8
    dyv = torch.randn(n, co, D, D, D, device=DEV)
    xv = torch.randn(n, ci, D, D, D, device=DEV) + 0.3
    w = torch.randn(co, ci, 3, 3, 3, device=DEV) / (ci * 27) ** 0.5
    gamma, beta = torch.randn(ci, device=DEV) * 0.3 + 1, torch.randn(ci, device=DEV) * 0.2
    dy, x = L.Act.from_ncdhw(dyv, split=split), L.Act.from_ncdhw(xv, split=split)
    wdh, wdl, _, _, _ = L.pack_weights(w, 1, split=split)
    _, _, _, _, wq = _packed_to_torch(L, w, 0, split, co, ci, 3)
    coef = torch.empty(n, ci, 4, device=DEV)
    L.gn_apply(x, L.Act.empty(n, D, D, D, ci, split=split), _channel_stats(x), gamma, beta, ci, G, coef)
    bst = torch.zeros(n, ci, 2, dtype=torch.float64, device=DEV)
    dz = L.Act.empty(n, D, D, D, ci, split=split)
    mode1 = dict(mode=1, gn_x=x, coef=coef, coef_ld=ci, bstats=bst)
    route = L.conv3d_route(dy, wdh, wdl, 3, 1, dz, ci, co, **mode1)
    assert (route["kind"], route["bn"], route["kc"]) == ("tap", 32, 64)
    L.conv3d(dy, wdh, wdl, 3, 1, dz, ci, co, **mode1)
    xq = x.to_ncdhw(ci).double().cpu().requires_grad_(True)
    z = F.group_norm(xq, G, gamma.double().cpu(), beta.double().cpu(), 1e-5)
    z.retain_grad()
    F.conv3d(F.relu(z), wq, padding=1).backward(dy.to_ncdhw(co).double().cpu())
    assert rel(dz.to_ncdhw(ci), z.grad) < TOL_STORE[split] * 1.5
    mu, rstd = coef[..., 2].double().cpu(), coef[..., 3].double().cpu()
    xhat = (xq.detach() - mu[:, :, None, None, None]) * rstd[:, :, None, None, None]
    b_ref = torch.stack([z.grad.sum(dim=(2, 3, 4)), (z.grad * xhat).sum(dim=(2, 3, 4))], dim=-1)
    assert rel(bst, b_ref) < 1e-4


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("ci,co,odims", [(32, 32, (8, 8, 8)), (64, 64, (4, 8, 16)), (128, 128, (4, 4, 8)), (16, 24, (3, 5, 6)),
                                         (32, 32, (16, 16, 16))])
@pytest.mark.parametrize("with_res", [False, True])
def test_stride2_data_gradient_by_parity_classes(pkg, ci, co, odims, with_res, split):
    """dX of a 3x3x3 stride-2 padding-1 convolution (encoder downsampling, myronenko.py:103-105) computed as eight
    parity-class implicit GEMMs over the un-inserted dY (cls_mode=1), (+ residual, * dropout scale), against autograd."""
    L = pkg.lib
    torch.manual_seed(ci + co + odims[0])
    n = 2
    idims = tuple(2 * d for d in odims)
    w = torch.randn(co, ci, 3, 3, 3, device=DEV) / (ci * 27) ** 0.5
    dy = L.Act.from_ncdhw(torch.randn(n, co, *odims, device=DEV), split=split)
    wdh, wdl, _, _, _ = L.pack_weights(w, 1, split=split)                 # [T][Cip][Cop], taps flipped
    _, _, cop, cip, wq = _packed_to_torch(L, w, 0, split, co, ci, 3)
    dx = L.Act.empty(n, *idims, cip, split=split, zero=True)
    res = L.Act.from_ncdhw(torch.randn(n, ci, *idims, device=DEV), split=split) if with_res else None
    scale = (torch.rand(n, cip, device=DEV) + 0.5) if with_res else None
    L.conv3d(dy, wdh, wdl, 3, 1, dx, cip, cop, res=res, scale=scale, cls_mode=1)
    xq = torch.zeros(n, ci, *idims, dtype=torch.float64, requires_grad=True)
    F.conv3d(xq, wq, stride=2, padding=1).backward(dy.to_ncdhw(co).double().cpu())
    ref = xq.grad
    if with_res:
        ref = (ref + res.to_ncdhw(ci).double().cpu()) * scale[:, :ci].double().cpu()[:, :, None, None, None]
    assert rel(dx.to_ncdhw(ci), ref) < TOL_STORE[split] * 1.5


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("ci,co,dims,ksz,stride", [
    (32, 32, (8, 8, 8), 3, 1), (64, 64, (8, 8, 8), 3, 1), (128, 128, (4, 8, 8), 3, 1), (256, 256, (4, 4, 8), 3, 1),
    (8, 32, (8, 8, 16), 3, 1), (16, 16, (8, 8, 8), 3, 1), (64, 32, (8, 8, 8), 3, 1), (24, 40, (5, 7, 9), 3, 1),
    (96, 192, (4, 4, 8), 3, 1), (256, 128, (4, 4, 8), 1, 1), (8, 32, (8, 8, 8), 1, 1), (32, 32, (16, 16, 16), 3, 2),
    (64, 64, (8, 8, 8), 3, 2),
    # 33..64 input channels with an output plane >= 8 x 16: the halo kernel of wgrad.cu in bf16 (the route is asserted)
    (64, 64, (4, 16, 8), 3, 1), (48, 32, (3, 18, 12), 3, 1), (40, 128, (2, 16, 16), 3, 1),
])
def test_conv3d_weight_gradient(pkg, ci, co, dims, ksz, stride, split):
    L = pkg.lib
    torch.manual_seed(ci + co)
    n = 2
    pad = ksz // 2
    od = [(s + 2 * pad - ksz) // stride + 1 for s in dims]
    a = L.Act.from_ncdhw(torch.randn(n, ci, *dims, device=DEV), split=split)
    dy = L.Act.from_ncdhw(torch.randn(n, co, *od, device=DEV), split=split)
    cip, cop, T = (ci + 7) // 8 * 8, (co + 7) // 8 * 8, ksz ** 3
    dw = torch.zeros(T, cip, cop, device=DEV)
    halo = not split and ksz == 3 and stride == 1 and 32 < ci <= 64 and od[1] >= 16 and od[2] >= 8
    assert L.wgrad_route(a, dy, ksz, stride, cip, cop)["kind"] == ("halo" if halo else "simt" if ksz == 1 and ci <= 16 else "tap")
    L.conv3d_wgrad(a, dy, ksz, stride, cip, cop, dw)
    out = torch.empty(co, ci, ksz, ksz, ksz, device=DEV)
    L.check(L.load_library().b200unet_unpack_wgrad(dw.data_ptr(), co, ci, cop, cip, T, 0, out.data_ptr(), L.stream_ptr()))
    wz = torch.zeros(co, ci, ksz, ksz, ksz, dtype=torch.float64, requires_grad=True)
    F.conv3d(a.to_ncdhw(ci).double().cpu(), wz, stride=stride, padding=pad).backward(dy.to_ncdhw(co).double().cpu())
    assert rel(out, wz.grad) < (1e-5 if not split else 5e-5)


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("C,G,dims", [(16, 8, (8, 12, 8)), (8, 8, (4, 4, 4)), (24, 24, (6, 4, 10)), (64, 8, (4, 4, 8)),
                                      (4, 4, (5, 6, 7))])   # 4 real channels in an 8-channel view: the network's first norm
def test_fused_groupnorm_relu_forward_backward(pkg, C, G, dims, split):
    """The kernels every norm layer of the plans launches: statistics -> coefficients -> GroupNorm + ReLU in one launch, and
    backward statistics -> dgamma, dbeta, dx in one launch; plus the first block's gn_bwd_finalize."""
    L = pkg.lib
    torch.manual_seed(C)
    n = 2
    S = dims[0] * dims[1] * dims[2]
    x = L.Act.from_ncdhw(torch.randn(n, C, *dims, device=DEV) * 2 + 0.5, split=split)
    Cv = x.c                                                 # view channels (C padded to 8): pitch of stats, coef, bstats
    gamma, beta = torch.randn(C, device=DEV) * 0.3 + 1, torch.randn(C, device=DEV) * 0.2
    stats = _channel_stats(x)
    stats[:, C:] = 7.0                                       # padded channels: ignored
    coef = torch.full((n, Cv, 4), float("nan"), device=DEV)  # every entry is written
    y = L.Act.empty(n, *dims, Cv, split=split)
    L.gn_apply(x, y, stats, gamma, beta, C, G, coef)
    xv = x.to_ncdhw(C).double().cpu()
    ref_np = np.maximum(group_norm(xv.numpy(), G, gamma.double().cpu().numpy(), beta.double().cpu().numpy()), 0)   # numpy oracle
    assert rel(y.to_ncdhw(C), torch.from_numpy(ref_np)) < TOL_STORE[split]
    xg = xv.reshape(n, G, -1)
    mu_ref = xg.mean(-1).repeat_interleave(C // G, dim=1)
    rstd_ref = (xg.var(-1, unbiased=False) + 1e-5).rsqrt().repeat_interleave(C // G, dim=1)
    a_ref = gamma.double().cpu() * rstd_ref
    assert rel(coef[:, :C, 2], mu_ref) < 1e-6 and rel(coef[:, :C, 3], rstd_ref) < 1e-6
    assert rel(coef[:, :C, 0], a_ref) < 1e-6 and rel(coef[:, :C, 1], beta.double().cpu() - mu_ref * a_ref) < 1e-6
    if Cv > C:
        assert float(coef[:, C:].abs().max()) == 0.0 and float(y.value()[..., C:].abs().max()) == 0.0
    # backward: dx = dL/dx given dz = dL/d(GN output)
    dz = L.Act.from_ncdhw(torch.randn(n, C, *dims, device=DEV), split=split)
    dzq = dz.to_ncdhw(C).double().cpu()
    xq = xv.clone().requires_grad_(True)
    g64, b64 = gamma.double().cpu().requires_grad_(True), beta.double().cpu().requires_grad_(True)
    F.group_norm(xq, G, g64, b64, 1e-5).backward(dzq)
    mu, rstd = coef[:, :C, 2].double().cpu(), coef[:, :C, 3].double().cpu()
    xhat = (xv - mu[:, :, None, None, None]) * rstd[:, :, None, None, None]
    bst = torch.zeros(n, Cv, 2, dtype=torch.float64)
    bst[:, :C] = torch.stack([dzq.sum(dim=(2, 3, 4)), (dzq * xhat).sum(dim=(2, 3, 4))], dim=-1)
    bst = bst.to(DEV)
    add = L.Act.from_ncdhw(torch.randn(n, C, *dims, device=DEV), split=split)
    dx = L.Act.empty(n, *dims, Cv, split=split)
    dg, db = torch.full((C,), float("nan"), device=DEV), torch.full((C,), float("nan"), device=DEV)
    L.gn_bwd(dz, x, coef, bst, gamma, C, G, dx, dg, db, add1=add)
    assert rel(dx.to_ncdhw(C), xq.grad + add.to_ncdhw(C).double().cpu()) < TOL_STORE[split]
    assert rel(dg, g64.grad) < 1e-5 and rel(db, b64.grad) < 1e-5
    if Cv > C:
        assert float(dx.value()[..., C:].abs().max()) == 0.0      # A = E = F = 0, and the padded add channels are zero
    # the first block's norm: (E, F) of dx = A dz + E x + F for the input gradient, dgamma and dbeta
    coef2 = torch.full((n, Cv, 2), float("nan"), device=DEV)
    dg2, db2 = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
    L.gn_bwd_finalize(bst, coef, gamma, n, C, Cv, G, S, coef2, dg2, db2)
    k, e = coef[:, :C].double().cpu(), coef2[:, :C].double().cpu()
    dx2 = k[..., 0, None, None, None] * dzq + e[..., 0, None, None, None] * xv + e[..., 1, None, None, None]
    assert rel(dx2, xq.grad) < TOL_STORE[True]
    assert rel(dg2, g64.grad) < 1e-5 and rel(db2, b64.grad) < 1e-5
    if Cv > C:
        assert float(coef2[:, C:].abs().max()) == 0.0


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("dims", [(4, 6, 8), (3, 5, 7), (1, 2, 4), (2, 2, 6)])   # even extents: register-blocked adjoint; (2, ..): first == last block
def test_trilinear_upsample_forward_backward(pkg, dims, split):
    L = pkg.lib
    torch.manual_seed(5)
    n, C = 2, 16
    x = L.Act.from_ncdhw(torch.randn(n, C, *dims, device=DEV), split=split)
    od = [2 * s for s in dims]
    cat = L.Act.empty(n, *od, 2 * C, split=split, zero=True)
    stats = torch.zeros(n, 2 * C, 2, dtype=torch.float64, device=DEV)
    L.upsample2x_fwd(x, cat.slice(0, C), stats, 2 * C)
    ref = trilinear_upsample2x(x.to_ncdhw(C).double().cpu().numpy())                     # numpy oracle
    got = cat.slice(0, C).to_ncdhw(C)
    assert rel(got, torch.from_numpy(ref)) < TOL_STORE[split]
    assert float(cat.hi[..., C:].float().abs().max()) == 0.0
    gd = torch.from_numpy(ref)
    s_ref = torch.stack([gd.sum(dim=(2, 3, 4)), (gd * gd).sum(dim=(2, 3, 4))], dim=-1)
    assert rel(stats[:, :C], s_ref) < 1e-5
    dy = L.Act.from_ncdhw(torch.randn(n, C, *od, device=DEV), split=split)
    dx = L.Act.empty(n, *dims, C, split=split)
    L.upsample2x_bwd(dy, dx)
    xq = x.to_ncdhw(C).double().cpu().requires_grad_(True)
    F.interpolate(xq, scale_factor=2, mode="trilinear", align_corners=False).backward(dy.to_ncdhw(C).double().cpu())
    assert rel(dx.to_ncdhw(C), xq.grad) < TOL_STORE[split]


@pytest.mark.parametrize("split", [False, True])
def test_head_forward_backward(pkg, split):
    L = pkg.lib
    torch.manual_seed(6)
    n, C, O, dims = 2, 32, 3, (6, 6, 10)
    x = L.Act.from_ncdhw(torch.randn(n, C, *dims, device=DEV), split=split)
    w = torch.randn(O, C, device=DEV) * 0.3
    logits = torch.empty(n, O, *dims, device=DEV)
    L.head_fwd(x, w, O, 0, logits)
    xv = x.to_ncdhw(C).double().cpu()
    assert rel(logits, torch.einsum("ncdhw,oc->nodhw", xv, w.double().cpu())) < 1e-6
    dl = torch.randn(n, O, *dims, device=DEV)
    dx = L.Act.empty(n, *dims, C, split=split)
    dw = torch.empty(O, C, device=DEV)
    L.head_bwd(x, w, O, dl, dx, dw)
    assert rel(dx.to_ncdhw(C), torch.einsum("nodhw,oc->ncdhw", dl.double().cpu(), w.double().cpu())) < TOL_STORE[split]
    assert rel(dw, torch.einsum("nodhw,ncdhw->oc", dl.double().cpu(), xv)) < 1e-5


@pytest.mark.parametrize("kw", [dict(sigmoid=True), dict(sigmoid=True, squared_pred=True), dict(sigmoid=True, jaccard=True),
                                dict(sigmoid=True, batch=True), dict(sigmoid=True, include_background=False),
                                dict(sigmoid=False), dict(sigmoid=True, reduction="sum")])
@pytest.mark.parametrize("dims", [(12, 10, 16), (5, 7, 3)])
def test_dice_forward_backward(pkg, kw, dims):
    torch.manual_seed(7)
    n, C = 2, 3
    x = torch.randn(n, C, *dims, device=DEV)
    t = (torch.rand(n, C, *dims, device=DEV) > 0.7).to(torch.uint8)
    crit = pkg.DiceLoss(**kw)
    xq = x.clone().requires_grad_(True)
    loss = crit(xq, t)
    loss.backward()
    xr = x.double().cpu().requires_grad_(True)
    lr = dice_loss(xr, t.cpu(), **{"sigmoid": False, **kw})
    lr.backward()
    assert abs(float(loss) - float(lr)) < 1e-6
    assert rel(xq.grad, xr.grad) < 1e-5


def test_dice_edge_cases(pkg):
    crit = pkg.DiceLoss(sigmoid=True)
    z = torch.zeros(1, 2, 4, 4, 4, device=DEV)
    t0 = torch.zeros(1, 2, 4, 4, 4, dtype=torch.uint8, device=DEV)
    # empty target: f = 1 - nr/(P + dr) with P = 32
    assert abs(float(crit(z, t0)) - (1 - 1e-5 / (32 + 1e-5))) < 1e-6
    with pytest.raises(AssertionError):
        crit(z, t0[:, :1])


def _packed_layout(w, mode, cop, cip):
    """fp32 restatement of a packed weight (kernels.h PackJob.mode), zero padded to (cop, cip)"""
    if mode >= 2:                                   # ConvTranspose3d weight [Ci][Co][k^3]
        w = w.transpose(0, 1)
    co, ci = w.shape[:2]
    t = w.reshape(co, ci, -1)
    if mode in (1, 2):                              # taps flipped
        t = t.flip(2)
    out = torch.zeros(t.shape[2], cop, cip)
    out[:, :co, :ci] = t.permute(2, 0, 1)
    return out.transpose(1, 2) if mode in (1, 3) else out   # data-gradient layouts: [T][Cip][Cop]


def test_weight_pack_unpack_roundtrip(pkg):
    L = pkg.lib
    torch.manual_seed(8)
    w = torch.randn(24, 12, 3, 3, 3, device=DEV)
    hi, lo, cop, cip, T = L.pack_weights(w, 0, split=True, cip=16)
    assert (cop, cip, T) == (24, 16, 27)
    assert rel((hi.float() + lo.float())[:, :24, :12], w.permute(2, 3, 4, 0, 1).reshape(27, 24, 12)) < 1e-5
    assert float(hi[:, :, 12:].float().abs().max()) == 0.0
    hi, lo, _, _, _ = L.pack_weights(w, 1, split=True, cip=16)
    assert rel((hi.float() + lo.float())[:, :12, :24], w.flip(2, 3, 4).permute(2, 3, 4, 1, 0).reshape(27, 12, 24)) < 1e-5
    # packed bits: hi and lo round to nearest even, exactly as torch's own conversion does
    for shape, modes in [((24, 12, 3, 3, 3), range(5)),
                         ((320, 256, 3, 3, 3), (0, 1)),      # more 16 x 16 tiles than blocks
                         ((16, 8, 2, 2, 2), (3, 4)),         # T = 8 ConvTranspose3d weight [Ci][Co][2][2][2]
                         ((40, 12, 1, 1, 1), (0, 1))]:       # T = 1
        w = torch.randn(*shape, device=DEV)
        for mode in modes:
            hi, lo, cop, cip, _ = L.pack_weights(w, mode, split=True)
            ref = _packed_layout(w.cpu(), mode, cop, cip)
            ref_hi = ref.bfloat16()
            assert torch.equal(hi.cpu(), ref_hi), (shape, mode)
            assert torch.equal(lo.cpu(), (ref - ref_hi.float()).bfloat16()), (shape, mode)
    # unpacking is an exact copy: fp32 [T][Cip][Cop] -> [Co][Ci][T] (mode 0) or, taps flipped back, [Ci][Co][T] (mode 2)
    co, ci, cop, cip, T = 20, 12, 24, 16, 27
    g = torch.randn(T, cip, cop, device=DEV)
    for mode, ref in [(0, g[:, :ci, :co].permute(2, 1, 0)), (2, g.flip(0)[:, :ci, :co].permute(1, 2, 0))]:
        out = torch.empty(ref.shape, device=DEV)
        L.check(L.load_library().b200unet_unpack_wgrad(g.data_ptr(), co, ci, cop, cip, T, mode, out.data_ptr(), L.stream_ptr()))
        assert torch.equal(out, ref.contiguous()), mode
    # the packed layouts are written in 8-channel chunks
    with pytest.raises(RuntimeError, match="multiples of 8"):
        L.pack_weights(w, 0, cip=12)


def test_errors_are_loud(pkg):
    L = pkg.lib
    a = L.Act.empty(1, 4, 4, 4, 8)
    y = L.Act.empty(1, 5, 4, 4, 8)                       # wrong output extent
    w = torch.zeros(27, 8, 8, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="do not produce output"):
        L.conv3d(a, w, None, 3, 1, y, 8, 8)
    with pytest.raises(RuntimeError, match="kernel_size"):
        L.conv3d(a, w, None, 5, 1, a, 8, 8)
