"""On-GPU diagnostics: runs groups of kernel checks and prints error magnitudes (does not assert -- it is the
bring-up tool; the pass/fail parity tests live in tests/).  Usage: python tools/gpu_diag.py <group> [...]
Groups: elementwise conv wgrad model
References here are torch fp64 ops on the GPU (the pytest suite uses the CPU oracle)."""
import importlib
import json
import os
import sys
import time
import traceback

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dunetcnn_b200")
L = pkg.lib
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
DEV = "cuda"
RESULTS = {}


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def maxabs(a, b):
    return float((a.double() - b.double()).abs().max())


def report(name, **kw):
    RESULTS[name] = kw
    print("[diag] %-58s %s" % (name, "  ".join("%s=%.3e" % (k, v) if isinstance(v, float) else "%s=%s" % (k, v) for k, v in kw.items())), flush=True)


def run(name, fn):
    try:
        fn()
        torch.cuda.synchronize()
    except Exception as e:  # noqa
        print("[diag] %-58s EXCEPTION %s" % (name, repr(e)[:400]), flush=True)
        traceback.print_exc()
        RESULTS[name] = {"exception": repr(e)[:400]}


def bf16r(x):
    return x.to(torch.bfloat16).float()


# ---------------------------------------------------------------------------------------------- elementwise
def group_elementwise():
    torch.manual_seed(0)
    for split in (False, True):
        tag = " split" if split else ""

        def t_roundtrip():
            x = torch.randn(2, 12, 6, 10, 8, device=DEV)
            a = L.Act.from_ncdhw(x, split=split)
            y = a.to_ncdhw(12)
            report("layout roundtrip" + tag, rel=rel(y, x), pad_zero=float(a.hi[..., 12:].float().abs().max()))
        run("layout roundtrip" + tag, t_roundtrip)

        def t_gn():
            N, Cc, D, H, W, G = 2, 16, 8, 12, 8, 8
            x = torch.randn(N, Cc, D, H, W, device=DEV) * 2 + 0.5
            gamma = torch.randn(Cc, device=DEV) * 0.3 + 1
            beta = torch.randn(Cc, device=DEV) * 0.2
            a = L.Act.from_ncdhw(x, split=split)
            xv = a.to_ncdhw(Cc).double()
            stats = torch.zeros(N, Cc, 2, dtype=torch.float64, device=DEV)
            L.channel_stats(a, stats, Cc)
            s_ref = torch.stack([xv.sum(dim=(2, 3, 4)), (xv * xv).sum(dim=(2, 3, 4))], dim=-1)
            coef = torch.empty(N, Cc, 4, device=DEV)
            L.gn_finalize(stats, gamma, beta, N, Cc, Cc, G, D * H * W, 1e-5, coef)
            y = L.Act.empty(N, D, H, W, Cc, split=split)
            L.gn_apply(a, y, coef, 0.0)
            ref = F.relu(F.group_norm(xv, G, gamma.double(), beta.double(), 1e-5))
            report("gn stats/apply" + tag, stats_rel=rel(stats, s_ref), y_rel=rel(y.to_ncdhw(Cc), ref))
            # backward
            dzv = torch.randn(N, Cc, D, H, W, device=DEV)
            dz = L.Act.from_ncdhw(dzv, split=split)
            dzq = dz.to_ncdhw(Cc).double()
            xq = xv.clone().requires_grad_(True)
            g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
            z = F.group_norm(xq, G, g64, b64, 1e-5)
            z.backward(dzq)
            mu, rstd = coef[..., 2].double(), coef[..., 3].double()
            xhat = (xv - mu[:, :, None, None, None]) * rstd[:, :, None, None, None]
            bst = torch.stack([dzq.sum(dim=(2, 3, 4)), (dzq * xhat).sum(dim=(2, 3, 4))], dim=-1).contiguous()
            coef2 = torch.empty(N, Cc, 2, device=DEV)
            dg = torch.empty(Cc, device=DEV); db = torch.empty(Cc, device=DEV)
            L.gn_bwd_finalize(bst, coef, gamma, N, Cc, Cc, G, D * H * W, coef2, dg, db)
            dx = L.Act.empty(N, D, H, W, Cc, split=split)
            addv = torch.randn(N, Cc, D, H, W, device=DEV)
            add = L.Act.from_ncdhw(addv, split=split)
            L.gn_bwd(dz, a, coef, coef2, dx, add1=add)
            report("gn backward" + tag, dx_rel=rel(dx.to_ncdhw(Cc), xq.grad + add.to_ncdhw(Cc).double()),
                   dgamma_rel=rel(dg, g64.grad), dbeta_rel=rel(db, b64.grad))
        run("gn" + tag, t_gn)

        def t_up():
            N, Cc, D, H, W = 2, 16, 4, 6, 8
            x = torch.randn(N, Cc, D, H, W, device=DEV)
            a = L.Act.from_ncdhw(x, split=split)
            cat = L.Act.empty(N, 2 * D, 2 * H, 2 * W, 2 * Cc, split=split, zero=True)
            stats = torch.zeros(N, 2 * Cc, 2, dtype=torch.float64, device=DEV)
            L.upsample2x_fwd(a, cat.slice(0, Cc), stats, 2 * Cc)
            ref = F.interpolate(a.to_ncdhw(Cc).double(), scale_factor=2, mode="trilinear", align_corners=False)
            got = cat.slice(0, Cc).to_ncdhw(Cc)
            s_ref = torch.stack([got.double().sum(dim=(2, 3, 4)), (got.double() ** 2).sum(dim=(2, 3, 4))], dim=-1)
            report("upsample fwd" + tag, rel=rel(got, ref), stats_rel=rel(stats[:, :Cc], s_ref),
                   other_half=float(cat.hi[..., Cc:].float().abs().max()))
            dyv = torch.randn(N, Cc, 2 * D, 2 * H, 2 * W, device=DEV)
            dy = L.Act.from_ncdhw(dyv, split=split)
            dx = L.Act.empty(N, D, H, W, Cc, split=split)
            L.upsample2x_bwd(dy, dx)
            xq = a.to_ncdhw(Cc).double().requires_grad_(True)
            F.interpolate(xq, scale_factor=2, mode="trilinear", align_corners=False).backward(dy.to_ncdhw(Cc).double())
            report("upsample bwd" + tag, rel=rel(dx.to_ncdhw(Cc), xq.grad))
        run("upsample" + tag, t_up)

        def t_head():
            N, Cc, D, H, W, O = 2, 16, 6, 6, 10, 3
            x = torch.randn(N, Cc, D, H, W, device=DEV)
            w = torch.randn(O, Cc, device=DEV) * 0.3
            a = L.Act.from_ncdhw(x, split=split)
            logits = torch.empty(N, O, D, H, W, device=DEV)
            L.head_fwd(a, w, O, 0, logits)
            xv = a.to_ncdhw(Cc).double()
            ref = torch.einsum("ncdhw,oc->nodhw", xv, w.double())
            dl = torch.randn(N, O, D, H, W, device=DEV)
            dx = L.Act.empty(N, D, H, W, Cc, split=split)
            dw = torch.empty(O, Cc, device=DEV)
            L.head_bwd(a, w, O, dl, dx, dw)
            report("head fwd/bwd" + tag, fwd_rel=rel(logits, ref),
                   dx_rel=rel(dx.to_ncdhw(Cc), torch.einsum("nodhw,oc->ncdhw", dl.double(), w.double())),
                   dw_rel=rel(dw, torch.einsum("nodhw,ncdhw->oc", dl.double(), xv)))
        run("head" + tag, t_head)

    def t_dice():
        N, Cc, D, H, W = 2, 3, 12, 10, 16
        x = torch.randn(N, Cc, D, H, W, device=DEV)
        t = (torch.rand(N, Cc, D, H, W, device=DEV) > 0.7).to(torch.uint8)
        from oracle import dice_loss
        for kw in (dict(sigmoid=True), dict(sigmoid=True, squared_pred=True), dict(sigmoid=True, jaccard=True),
                   dict(sigmoid=True, batch=True), dict(sigmoid=True, include_background=False), dict(sigmoid=False)):
            crit = pkg.DiceLoss(**kw)
            xq = x.clone().requires_grad_(True)
            loss = crit(xq, t)
            loss.backward()
            xr = x.double().clone().requires_grad_(True)
            xin = xr if kw.get("sigmoid") else xr
            lr = dice_loss(xin, t, **{"sigmoid": False, **kw})
            lr.backward()
            report("dice %s" % kw, loss_abs=abs(float(loss) - float(lr)), grad_rel=rel(xq.grad, xr.grad))
    run("dice", t_dice)

    def t_pack():
        w = torch.randn(24, 12, 3, 3, 3, device=DEV)
        hi, lo, cop, cip, T = L.pack_weights(w, 0, split=True, cip=16)
        got = (hi.float() + lo.float())[:, :24, :12]
        report("pack fwd", rel=rel(got, w.permute(2, 3, 4, 0, 1).reshape(27, 24, 12)), pad=float(hi[:, :, 12:].float().abs().max()))
        hi, lo, cop, cip, T = L.pack_weights(w, 1, split=True, cip=16)
        got = (hi.float() + lo.float())[:, :12, :24]
        report("pack dgrad", rel=rel(got, w.flip(2, 3, 4).permute(2, 3, 4, 1, 0).reshape(27, 12, 24)))
    run("pack", t_pack)


# ---------------------------------------------------------------------------------------------- conv
def conv_case(cin, cout, dims, ksz, stride, split, n=2, extras=False):
    torch.manual_seed(cin * 1000 + cout + ksz)
    D, H, W = dims
    x = torch.randn(n, cin, D, H, W, device=DEV)
    w = torch.randn(cout, cin, ksz, ksz, ksz, device=DEV) / (cin * ksz ** 3) ** 0.5
    a = L.Act.from_ncdhw(x, split=split)
    whi, wlo, cop, cip, T = L.pack_weights(w, 0, split=split)
    pad = ksz // 2
    Do, Ho, Wo = [(s + 2 * pad - ksz) // stride + 1 for s in dims]
    y = L.Act.empty(n, Do, Ho, Wo, cop, split=split, zero=True)
    xq = a.to_ncdhw(cin).double()
    wq = (whi.float() + (wlo.float() if split else 0)).double()[:, :cout, :cin].reshape(ksz, ksz, ksz, cout, cin).permute(3, 4, 0, 1, 2)
    ref = F.conv3d(xq, wq, stride=stride, padding=pad)
    kw = {}
    res = scale = stats = None
    if extras:
        resv = torch.randn(n, cout, Do, Ho, Wo, device=DEV)
        res = L.Act.from_ncdhw(resv, split=split)
        scale = ((torch.rand(n, cop, device=DEV) > 0.3).float() * 1.25).contiguous()
        stats = torch.zeros(n, cop, 2, dtype=torch.float64, device=DEV)
        kw = dict(res=res, scale=scale, stats=stats, stats_ld=cop)
        ref = (ref + res.to_ncdhw(cout).double()) * scale[:, :cout, None, None, None].double()
    t0 = time.time()
    L.conv3d(a, whi, wlo, ksz, stride, y, cop, cip, **kw)
    torch.cuda.synchronize()
    got = y.to_ncdhw(cout)
    ys = L.Act.empty(n, Do, Ho, Wo, cop, split=split, zero=True)
    out = dict(rel=rel(got, ref), maxabs=maxabs(got, ref), refmax=float(ref.abs().max()))
    if not extras and cin * cout * D * H * W * n <= 64 * 64 * 16 ** 3 * 2:
        L.conv3d_simt(a, whi, wlo, ksz, stride, ys)
        out["rel_vs_simt"] = rel(got, ys.to_ncdhw(cout))
        out["simt_vs_ref"] = rel(ys.to_ncdhw(cout), ref)
    if extras:
        gd = got.double()
        s_ref = torch.stack([gd.sum(dim=(2, 3, 4)), (gd * gd).sum(dim=(2, 3, 4))], dim=-1)
        out["stats_rel"] = rel(stats[:, :cout], s_ref)
    report("conv ci%d co%d %s k%d s%d%s%s" % (cin, cout, "x".join(map(str, dims)), ksz, stride, " split" if split else "",
                                              " +res/scale/stats" if extras else ""), **out)


def group_conv():
    cases = [
        (64, 64, (8, 8, 8), 3, 1, False), (32, 32, (8, 8, 16), 3, 1, False), (16, 16, (8, 8, 8), 3, 1, False),
        (8, 8, (8, 8, 8), 3, 1, False), (8, 32, (16, 16, 16), 3, 1, False), (128, 128, (8, 8, 8), 3, 1, False),
        (256, 256, (4, 4, 8), 3, 1, False), (64, 32, (8, 12, 8), 3, 1, False), (24, 40, (6, 10, 12), 3, 1, False),
        (96, 192, (4, 4, 8), 3, 1, False), (64, 128, (8, 8, 8), 1, 1, False), (256, 128, (4, 4, 8), 1, 1, False),
        (32, 32, (16, 16, 16), 3, 2, False), (64, 64, (8, 8, 8), 3, 2, False), (8, 8, (8, 8, 8), 3, 2, False),
        (32, 32, (5, 7, 9), 3, 1, False),
        # halo mode of the convolution kernel (output plane >= 8 x 16)
        (32, 32, (8, 16, 16), 3, 1, False), (64, 32, (4, 16, 8), 3, 1, False), (8, 32, (16, 16, 16), 3, 1, False),
        (128, 128, (8, 16, 8), 3, 1, False), (256, 256, (2, 16, 8), 3, 1, False), (24, 40, (6, 18, 12), 3, 1, False),
        (96, 192, (3, 16, 8), 3, 1, False), (32, 64, (5, 24, 20), 3, 1, False), (16, 16, (1, 16, 8), 3, 1, False),
        (32, 32, (8, 16, 16), 3, 1, True), (128, 128, (4, 16, 8), 3, 1, True),
        (64, 64, (8, 8, 8), 3, 1, True), (32, 64, (8, 8, 8), 3, 1, True), (8, 8, (8, 8, 8), 3, 1, True),
        (32, 32, (8, 8, 8), 3, 2, True),
    ]
    for c in cases:
        run("conv %s" % (c,), lambda c=c: conv_case(*c))
    for c in [(32, 32, (8, 8, 8), 3, 1, False), (64, 128, (8, 8, 8), 3, 1, True), (32, 32, (8, 16, 16), 3, 1, False),
              (64, 128, (4, 16, 16), 3, 1, True)]:
        run("conv extras %s" % (c,), lambda c=c: conv_case(*c, extras=True))

    def t_two_src():
        for split in (False, True):
            n, ci, co, D = 2, 8, 32, 8
            x = torch.randn(n, ci, D, D, D, device=DEV)
            h = torch.randn(n, co, D, D, D, device=DEV)
            w2 = torch.randn(co, co, 3, 3, 3, device=DEV) / (co * 27) ** 0.5
            ws = torch.randn(co, ci, 1, 1, 1, device=DEV) / ci ** 0.5
            ax, ah = L.Act.from_ncdhw(x, split=split), L.Act.from_ncdhw(h, split=split)
            w2h, w2l, cop, cip, _ = L.pack_weights(w2, 0, split=split)
            wsh, wsl, _, cips, _ = L.pack_weights(ws, 0, split=split)
            y = L.Act.empty(n, D, D, D, co, split=split)
            L.conv3d(ah, w2h, w2l, 3, 1, y, cop, cip, x2=ax, w2_hi=wsh, w2_lo=wsl, cip2=cips)
            w2q = (w2h.float() + (w2l.float() if split else 0)).double().reshape(3, 3, 3, co, co).permute(3, 4, 0, 1, 2)
            wsq = (wsh.float() + (wsl.float() if split else 0)).double()[:, :co, :ci].reshape(1, 1, 1, co, ci).permute(3, 4, 0, 1, 2)
            ref = F.conv3d(ah.to_ncdhw(co).double(), w2q, padding=1) + F.conv3d(ax.to_ncdhw(ci).double(), wsq)
            report("conv two-source%s" % (" split" if split else ""), rel=rel(y.to_ncdhw(co), ref))
    run("conv two-source", t_two_src)

    def t_mode1():
        for split in (False, True):
            n, ci, co, D, G = 2, 32, 32, 8, 8
            dyv = torch.randn(n, co, D, D, D, device=DEV)
            xv = torch.randn(n, ci, D, D, D, device=DEV) + 0.3
            w = torch.randn(co, ci, 3, 3, 3, device=DEV) / (ci * 27) ** 0.5
            gamma = torch.randn(ci, device=DEV) * 0.3 + 1
            beta = torch.randn(ci, device=DEV) * 0.2
            dy, x = L.Act.from_ncdhw(dyv, split=split), L.Act.from_ncdhw(xv, split=split)
            wdh, wdl, cop_rows, cip_k, _ = L.pack_weights(w, 1, split=split)   # [T][ci][co]
            stats = torch.zeros(n, ci, 2, dtype=torch.float64, device=DEV)
            L.channel_stats(x, stats, ci)
            coef = torch.empty(n, ci, 4, device=DEV)
            L.gn_finalize(stats, gamma, beta, n, ci, ci, G, D ** 3, 1e-5, coef)
            bst = torch.zeros(n, ci, 2, dtype=torch.float64, device=DEV)
            dz = L.Act.empty(n, D, D, D, ci, split=split)
            # weights for dgrad: rows = ci (cip of original), K = co (cop of original)
            L.conv3d(dy, wdh, wdl, 3, 1, dz, (ci + 7) // 8 * 8, (co + 7) // 8 * 8, mode=1, gn_x=x, coef=coef, coef_ld=ci,
                     bstats=bst)
            xq = x.to_ncdhw(ci).double().requires_grad_(True)
            wq = (L.pack_weights(w, 0, split=split)[0].float() + (L.pack_weights(w, 0, split=split)[1].float() if split else 0)
                  ).double().reshape(3, 3, 3, co, ci).permute(3, 4, 0, 1, 2)
            z = F.group_norm(xq, G, gamma.double(), beta.double(), 1e-5)
            a = F.relu(z)
            a.retain_grad(); z.retain_grad()
            y = F.conv3d(a, wq, padding=1)
            y.backward(dy.to_ncdhw(co).double())
            dz_ref = z.grad
            mu, rstd = coef[..., 2].double(), coef[..., 3].double()
            xhat = (xq.detach() - mu[:, :, None, None, None]) * rstd[:, :, None, None, None]
            b_ref = torch.stack([dz_ref.sum(dim=(2, 3, 4)), (dz_ref * xhat).sum(dim=(2, 3, 4))], dim=-1)
            report("conv dgrad mode1%s" % (" split" if split else ""), dz_rel=rel(dz.to_ncdhw(ci), dz_ref), bstats_rel=rel(bst, b_ref))
    run("conv mode1", t_mode1)


def group_wgrad():
    cases = [(32, 32, (8, 8, 8), 3, 1, False), (64, 64, (8, 8, 8), 3, 1, False), (128, 128, (8, 8, 8), 3, 1, False),
             (256, 256, (4, 4, 8), 3, 1, False), (8, 32, (8, 8, 16), 3, 1, False), (16, 16, (8, 8, 8), 3, 1, False),
             (64, 32, (8, 8, 8), 3, 1, False), (24, 40, (6, 10, 12), 3, 1, False), (96, 192, (4, 4, 8), 3, 1, False),
             (256, 128, (4, 4, 8), 1, 1, False), (8, 32, (8, 8, 8), 1, 1, False), (32, 32, (16, 16, 16), 3, 2, False),
             (64, 64, (8, 8, 8), 3, 2, False),
             (32, 32, (8, 8, 8), 3, 1, True), (64, 128, (8, 8, 8), 3, 1, True), (32, 32, (8, 8, 8), 3, 2, True)]
    for (ci, co, dims, ksz, stride, split) in cases:
        def t(ci=ci, co=co, dims=dims, ksz=ksz, stride=stride, split=split):
            torch.manual_seed(ci + co)
            n = 2
            D, H, W = dims
            pad = ksz // 2
            Do, Ho, Wo = [(s + 2 * pad - ksz) // stride + 1 for s in dims]
            av = torch.randn(n, ci, D, H, W, device=DEV)
            dyv = torch.randn(n, co, Do, Ho, Wo, device=DEV)
            a, dy = L.Act.from_ncdhw(av, split=split), L.Act.from_ncdhw(dyv, split=split)
            cip, cop = (ci + 7) // 8 * 8, (co + 7) // 8 * 8
            T = ksz ** 3
            dw = torch.zeros(T, cip, cop, device=DEV)
            L.conv3d_wgrad(a, dy, ksz, stride, cip, cop, dw)
            out = torch.empty(co, ci, ksz, ksz, ksz, device=DEV)
            L.check(L.load_library().b200unet_unpack_wgrad(dw.data_ptr(), co, ci, cop, cip, T, 0, out.data_ptr(), L.stream_ptr()))
            aq = a.to_ncdhw(ci).double()
            wz = torch.zeros(co, ci, ksz, ksz, ksz, dtype=torch.float64, device=DEV, requires_grad=True)
            F.conv3d(aq, wz, stride=stride, padding=pad).backward(dy.to_ncdhw(co).double())
            report("wgrad ci%d co%d %s k%d s%d%s" % (ci, co, "x".join(map(str, dims)), ksz, stride, " split" if split else ""),
                   rel=rel(out, wz.grad), maxabs=maxabs(out, wz.grad), refmax=float(wz.grad.abs().max()))
        run("wgrad %s" % ((ci, co, dims, ksz, stride, split),), t)


def group_model():
    from oracle import UNetConfig, make_state_dict, unet3d_forward, dice_loss
    for (kw, shape, precision) in [
        (dict(n_features=4, n_outputs=3, base_width=8), (1, 4, 32, 32, 32), "split"),
        (dict(n_features=4, n_outputs=3, base_width=8), (1, 4, 32, 32, 32), "bf16"),
        (dict(n_features=4, n_outputs=3, base_width=16), (2, 4, 32, 32, 32), "split"),
        (dict(n_features=1, n_outputs=1, base_width=8, encoder_blocks=[1, 2, 2, 4, 4]), (1, 1, 32, 32, 32), "split"),
        (dict(n_features=4, n_outputs=3, base_width=32), (2, 4, 32, 32, 32), "bf16"),
        (dict(n_features=4, n_outputs=3, base_width=8, use_transposed_convolutions=True), (1, 4, 32, 32, 32), "split"),
        (dict(n_features=4, n_outputs=3, base_width=16, use_transposed_convolutions=True), (2, 4, 32, 32, 32), "bf16"),
    ]:
        def t(kw=kw, shape=shape, precision=precision):
            cfg = UNetConfig(**kw)
            sd = make_state_dict(cfg, seed=0)
            model = pkg.UNet3D(precision=precision, **kw).cuda()
            model.load_state_dict(sd, strict=True)
            g = torch.Generator().manual_seed(1)
            x = torch.randn(shape, generator=g)
            tgt = (torch.rand((shape[0], cfg.n_outputs) + tuple(shape[2:]), generator=torch.Generator().manual_seed(2)) > 0.7).to(torch.uint8)
            mask = ((torch.rand((shape[0], cfg.base_width), generator=torch.Generator().manual_seed(3)) >= 0.2).float() / 0.8)
            # reference: fp64 functional restatement on the GPU
            sd64 = {k: v.double().cuda().requires_grad_(True) for k, v in sd.items()}
            ref = unet3d_forward(sd64, x.double().cuda(), cfg, dropout_mask=mask.cuda())
            lref = dice_loss(ref, tgt.cuda())
            lref.backward()
            model.train()
            model.set_dropout_scale(mask)
            crit = pkg.DiceLoss(sigmoid=True)
            out = model(x.cuda())
            loss = crit(out, tgt.cuda())
            loss.backward()
            torch.cuda.synchronize()
            worst = 0.0
            worst_k = ""
            rels = {}
            for k, p in model.named_parameters():
                r = rel(p.grad, sd64[k].grad)
                rels[k] = r
                if r > worst:
                    worst, worst_k = r, k
            report("model %s %s %s" % (kw, shape, precision), logits_rel=rel(out, ref), dice_abs=abs(float(loss) - float(lref)),
                   worst_grad_rel=worst, worst_key=worst_k, median_grad_rel=float(torch.tensor(list(rels.values())).median()),
                   launches_fwd=model.launches_last_forward, launches_bwd=model.launches_last_backward)
            bad = sorted(rels.items(), key=lambda kv: -kv[1])[:8]
            print("        worst grads:", ["%s=%.2e" % kv for kv in bad], flush=True)
            model.eval()
            with torch.no_grad():
                oe = model(x.cuda())
                re = unet3d_forward({k: v.detach() for k, v in sd64.items()}, x.double().cuda(), cfg)
            report("model eval %s %s" % (shape, precision), logits_rel=rel(oe, re))
        run("model %s %s" % (kw, precision), t)


def group_bench():
    for (kw, shape, precision) in [(dict(n_features=4, n_outputs=3, base_width=32), (2, 4, 128, 128, 128), "bf16"),
                                   (dict(n_features=4, n_outputs=3, base_width=32), (1, 4, 64, 64, 64), "split")]:
        def t(kw=kw, shape=shape, precision=precision):
            model = pkg.UNet3D(precision=precision, **kw).cuda()
            crit = pkg.DiceLoss(sigmoid=True)
            x = torch.randn(shape, device=DEV)
            tgt = (torch.rand((shape[0], kw["n_outputs"]) + tuple(shape[2:]), device=DEV) > 0.7).to(torch.uint8)
            model.train()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            times = []
            for it in range(5):
                model.zero_grad(set_to_none=True)
                ev[0].record()
                out = model(x)
                ev[1].record()
                loss = crit(out, tgt)
                ev[2].record()
                loss.backward()
                ev[3].record()
                torch.cuda.synchronize()
                times.append((ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3])))
            f, d, b = times[-1]
            report("bench %s %s" % (shape, precision), fwd_ms=f, dice_ms=d, bwd_ms=b, vol_per_s=shape[0] / ((f + d + b) / 1e3),
                   loss=float(loss), mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30, all_ms=str([tuple(round(v, 2) for v in t) for t in times]))
        run("bench %s" % (shape,), t)


GROUPS = {"bench": group_bench, "elementwise": group_elementwise, "conv": group_conv, "wgrad": group_wgrad,
          "model": group_model}

if __name__ == "__main__":
    names = sys.argv[1:] or list(GROUPS)
    print("device:", torch.cuda.get_device_name(0), "lib version", L.load_library().b200unet_version(), flush=True)
    for nme in names:
        print("==== group", nme, flush=True)
        run("group " + nme, GROUPS[nme])
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "diag_%s.json" % "_".join(names)), "w") as f:
        json.dump(RESULTS, f, indent=1, default=str)
