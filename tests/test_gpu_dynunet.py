"""DynUNet-style blocks on the GPU (SURVEY.md section 8f rank 1): post-activation conv -> InstanceNorm -> LeakyReLU(0.01),
ConvTranspose3d kernel = stride = 2 up-sampling, biased output block, non-power-of-two filter counts -- forward, Dice and
all parameter gradients against the restated oracle (oracle/dynunet_oracle.py: PARITY UNPINNED, MONAI is absent) and the
kernels it adds against torch autograd."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dice_loss
from oracle.dynunet_oracle import make_dynunet_state_dict, dynunet_forward

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _kw(cin, cout, filters):
    L = len(filters)
    return dict(spatial_dims=3, in_channels=cin, out_channels=cout, kernel_size=[[3, 3, 3]] * L, strides=[[1, 1, 1]] + [[2, 2, 2]] * (L - 1),
                upsample_kernel_size=[[2, 2, 2]] * (L - 1), filters=filters)


def _rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30))


@pytest.mark.parametrize("cin,cout,filters,shape", [(4, 3, [8, 16, 24, 32], (1, 4, 32, 32, 32)), (1, 2, [16, 24, 48], (2, 1, 16, 32, 24)),
                                                    (4, 3, [32, 64, 96], (1, 4, 32, 32, 64))])
def test_dynunet_split_precision_matches_unpinned_oracle(pkg, cin, cout, filters, shape):
    sd = make_dynunet_state_dict(cin, cout, filters, seed=1)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(shape, generator=g)
    t = (torch.rand((shape[0], cout) + shape[2:], generator=g) > 0.7).to(torch.uint8)
    sd64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    ref = dynunet_forward(sd64, x.double(), len(filters))
    lref = dice_loss(ref, t)
    lref.backward()
    model = pkg.DynUNet(precision="split", **_kw(cin, cout, filters)).to(DEV)
    model.load_state_dict(sd, strict=True)
    model.train()
    out = model(x.to(DEV))
    loss = pkg.DiceLoss(sigmoid=True)(out, t.to(DEV))
    loss.backward()
    assert _rel(out.detach(), ref.detach()) < 1e-3
    assert abs(float(loss) - float(lref)) < 1e-3 * abs(float(lref))
    for k, p in model.named_parameters():
        r = sd64[k].grad
        gn, rn = float(p.grad.double().norm()), float(r.norm())
        assert abs(gn - rn) < 3e-2 * rn + 1e-12, (k, gn, rn)
        cos = float((p.grad.double().cpu() * r).sum() / (gn * rn + 1e-30))
        # norm gains / shifts of an instance norm over few voxels are sums with heavy cancellation: measured 0.9987 on a
        # 24-element tensor (8 x 16 x 12 voxels per channel); everything larger holds the 0.999 bar of the UNet3D tests
        assert cos > (0.995 if p.numel() <= 64 else 0.999), (k, cos)
    model.eval()
    with torch.no_grad():
        out_inf = model(x.to(DEV))                                       # forward-only plan
    assert _rel(out_inf, ref.detach()) < 1e-3


def test_dynunet_bf16_mode_dice_bound(pkg):
    cin, cout, filters, shape = 4, 3, [16, 32, 48, 64], (1, 4, 32, 32, 32)
    sd = make_dynunet_state_dict(cin, cout, filters, seed=2)
    g = torch.Generator().manual_seed(6)
    x = torch.randn(shape, generator=g)
    t = (torch.rand((1, cout) + shape[2:], generator=g) > 0.7).to(torch.uint8)
    ref = dynunet_forward({k: v.double() for k, v in sd.items()}, x.double(), len(filters))
    model = pkg.DynUNet(precision="bf16", **_kw(cin, cout, filters)).to(DEV)
    model.load_state_dict(sd)
    model.train()
    out = model(x.to(DEV))
    loss = pkg.DiceLoss(sigmoid=True)(out, t.to(DEV))
    loss.backward()
    assert abs(float(loss) - float(dice_loss(ref, t))) < 1e-3
    assert _rel(out.detach(), ref) < 5e-2
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("ci,co,dims", [(32, 16, (4, 8, 8)), (96, 64, (4, 4, 8)), (24, 40, (3, 5, 6))])
def test_transposed_conv_k2s2_forward_dgrad_wgrad(pkg, ci, co, dims, split):
    """ConvTranspose3d(kernel = stride = 2): forward by parity classes (cls_mode 2), its data gradient (kernel-2 stride-2
    unpadded conv) and its weight gradient (roles swapped) against torch autograd."""
    L = pkg.lib
    torch.manual_seed(ci + co)
    n = 2
    odims = tuple(2 * d for d in dims)
    w = torch.randn(ci, co, 2, 2, 2, device=DEV) / (ci * 8) ** 0.5
    x = L.Act.from_ncdhw(torch.randn(n, ci, *dims, device=DEV), split=split)
    tol = 4e-3 if not split else 5e-5
    # forward: mode-4 pack [8][Cop][Cip]
    whi, wlo, cop, cip, _ = L.pack_weights(w, 4, split=split)
    wq = (whi.float() + (wlo.float() if split else 0)).double().cpu()[:, :co, :ci].reshape(2, 2, 2, co, ci).permute(4, 3, 0, 1, 2)
    y = L.Act.empty(n, *odims, cop, split=split, zero=True)
    L.conv3d(x, whi, wlo, 2, 1, y, cop, cip, cls_mode=2)
    xq = x.to_ncdhw(ci).double().cpu().requires_grad_(True)
    wq = wq.clone().requires_grad_(True)
    ref = F.conv_transpose3d(xq, wq, stride=2)
    assert _rel(y.to_ncdhw(co), ref.detach()) < tol
    # backward
    dy = L.Act.from_ncdhw(torch.randn(n, co, *odims, device=DEV), split=split)
    ref.backward(dy.to_ncdhw(co).double().cpu())
    wdh, wdl, _, _, _ = L.pack_weights(w, 3, split=split)                 # [8][Cip][Cop]
    dx = L.Act.empty(n, *dims, cip, split=split, zero=True)
    L.conv3d(dy, wdh, wdl, 2, 2, dx, cip, cop)
    assert _rel(dx.to_ncdhw(ci), xq.grad) < tol * 1.5
    dw = torch.zeros(8, cop, cip, device=DEV)                            # roles swapped: rows = co, columns = ci
    L.conv3d_wgrad(dy, x, 2, 2, cop, cip, dw)
    got = dw[:, :co, :ci].double().cpu().reshape(2, 2, 2, co, ci).permute(4, 3, 0, 1, 2)
    assert _rel(got, wq.grad) < (2e-3 if not split else 5e-5)


@pytest.mark.parametrize("split", [False, True])
def test_activation_backward_kernel_on_fused_coefficients(pkg, split):
    """dz = (g1 + g2) * LeakyReLU'(A c + B) with (sum dz, sum dz*xhat): through head-less plumbing = compare with autograd of
    LeakyReLU(InstanceNorm(c)) for the statistics and the mask."""
    import ctypes as C
    L = pkg.lib
    lib = L.load_library()
    torch.manual_seed(3)
    n, ch, dims = 2, 24, (6, 10, 8)
    c = L.Act.from_ncdhw(torch.randn(n, ch, *dims, device=DEV) * 2 + 0.5, split=split)
    g1 = L.Act.from_ncdhw(torch.randn(n, ch, *dims, device=DEV), split=split)
    g2 = L.Act.from_ncdhw(torch.randn(n, ch, *dims, device=DEV), split=split)
    gamma, beta = torch.randn(ch, device=DEV) * 0.3 + 1, torch.randn(ch, device=DEV) * 0.2
    cv = c.value().double()
    stats = torch.stack([cv.sum(dim=(1, 2, 3)), (cv * cv).sum(dim=(1, 2, 3))], dim=-1).contiguous()   # fp64 (sum, sumsq)
    coef = torch.empty(n, ch, 4, device=DEV)
    L.gn_apply(c, L.Act.empty(n, *dims, ch, split=split), stats, gamma, beta, ch, ch, coef, slope=0.01)   # G = C: instance norm
    dz = L.Act.empty(n, *dims, ch, split=split)
    bst = torch.zeros(n, ch, 2, dtype=torch.float64, device=DEV)
    g2t = g2.ct()
    L.check(lib.b200unet_act_bwd(C.byref(g1.ct()), C.byref(g2t), C.byref(c.ct()), coef.data_ptr(), C.c_float(0.01), C.byref(dz.ct()),
                                 bst.data_ptr(), ch, L.stream_ptr()), "act_bwd")
    cq = c.to_ncdhw(ch).double().cpu().requires_grad_(True)
    z = F.instance_norm(cq, weight=gamma.double().cpu(), bias=beta.double().cpu(), eps=1e-5)
    z.retain_grad()
    F.leaky_relu(z, 0.01).backward((g1.to_ncdhw(ch) + g2.to_ncdhw(ch)).double().cpu())
    assert _rel(dz.to_ncdhw(ch), z.grad) < (4e-3 if not split else 5e-5)
    mu, rstd = coef[..., 2].double().cpu(), coef[..., 3].double().cpu()
    xhat = (cq.detach() - mu[:, :, None, None, None]) * rstd[:, :, None, None, None]
    b_ref = torch.stack([z.grad.sum(dim=(2, 3, 4)), (z.grad * xhat).sum(dim=(2, 3, 4))], dim=-1)
    assert _rel(bst, b_ref) < 1e-4
