"""The Dice (csrc/dice.cu), Dice + cross-entropy (csrc/dice_ce.cu), sliding-window tiling and z-score (csrc/prepost.cu) kernels
against fp64, element by element, at the launch geometries of tests/loss_prepost_cases.py.

Every loss and every dlogit must satisfy |got - ref| <= bound, with the bound fixed by a model of the kernel's fp32 arithmetic,
never by what a GPU shows:
  - a sum a thread accumulates in fp32 over `chain` terms (the launch geometry gives it) is off by at most
    (chain + a few) * u * (the sum of the terms' absolute values), plus the terms' own error: the activated probability p has
    a relative error ep (sigmoid through __expf: (6 + 1.2 max|x|) u; softmax: (C + 6 + 4.5 max|x|) u; identity: 0);
  - the loss and the backward coefficients dF/dI, dF/dP move with those sums to first order; the coefficients are rounded to
    fp32 once;
  - every dlogit is the fp32 evaluation of its expression from the coefficients, each rounding bounded by u times the
    magnitudes it involves (for the sigmoid, 1 - p cancels, so p (1 - p) is off by (2 ep + 3 u) p).
u = 2^-24.  The fp64 references run on the device; on small cases the closed forms are checked against fp64 autograd first.
"""
import itertools
import time
import zlib

import pytest
import torch
import torch.nn.functional as F

import loss_prepost_cases as B

pytestmark = pytest.mark.gpu

DEV = "cuda"
f64 = torch.float64
U = B.U
U64 = 2.0 ** -53
GRAD_OUTS = (1.0, 0.37, -2.0)        # grad_out of the loss: (g * loss).backward() with g rounded to fp32
FULL_PRODUCT_MAX = 8 << 20           # cases up to this many logits run every flag combination; larger ones four of them
REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    t0 = time.time()
    yield
    print("\nobserved error as a fraction of its bound (worst over the case's flag combinations and elements):")
    for k, v in sorted(REPORT.items()):
        print("  %-75s %s" % (k, "  ".join("%s %.3f" % kv for kv in sorted(v.items()))))
    print("test_gpu_loss_prepost_kernels: %.1f s" % (time.time() - t0))


def note(case, what, frac):
    d = REPORT.setdefault(case.id, {})
    d[what] = max(d.get(what, 0.0), frac)


def gen_of(name):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(name.encode()))


def within(got, ref, lim, what):
    """|got - ref| <= lim at every element; returns the worst |got - ref| / lim, names the worst element on failure"""
    got = got.double()
    err = (got - ref).abs()
    bad = (err > lim) | ~torch.isfinite(got)
    if bool(bad.any()):
        worst = int(((err - lim).nan_to_num(float("inf")) * bad).flatten().argmax())
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), got.shape))
        pytest.fail("%s: %d of %d elements out of bounds; worst at %s: got %.10g ref %.10g bound %.3g"
                    % (what, int(bad.sum()), bad.numel(), idx, float(got[idx]), float(ref[idx]), float(lim[idx])))
    return float((err / lim.clamp_min(1e-300)).max()) if err.numel() else 0.0


def f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


# ---------------------------------------------------------------------------------------------- fp64 reference + bound
def act_error(act, C, X):
    """relative error bound of the kernel's fp32 p = act(x), |x| <= X"""
    if act == "sigmoid":
        return (6 + 1.2 * X) * U
    if act == "softmax":
        return (C + 6 + 4.5 * X) * U
    return 0.0


def reference(x, t, *, act, squared, jaccard, batch, include_background, reduction, lambda_dice=1.0, lambda_ce=0.0,
              with_ce=False, chain, soft_target, go, nr=1e-5, dr=1e-5):
    """x, t: [N, C, S] fp64 (t as the kernels see it: one-hot rows, a label map expanded, zero rows for labels outside [0, C)).
    Returns (loss, bound, dx, dx bound) for the kernels' Dice [+ CE] at grad_out go."""
    N, C, S = x.shape
    nr, dr, lambda_dice, lambda_ce = f32(nr), f32(dr), f32(lambda_dice), f32(lambda_ce)
    X = float(x.abs().max())
    ep = act_error(act, C, X)
    p = torch.sigmoid(x) if act == "sigmoid" else torch.softmax(x, 1) if act == "softmax" else x
    q = 2 * p if squared else torch.ones_like(p)
    c_lo = 1 if (not include_background and C > 1) else 0
    # per-(n, c) sums and their error: fp32 chains of `chain` terms, each term off by its p error and one product rounding
    I, AI = (p * t).sum(-1), (p * t).abs().sum(-1)
    P, AP = ((p * p).sum(-1), (p * p).sum(-1)) if squared else (p.sum(-1), p.abs().sum(-1))
    T, AT = ((t * t).sum(-1), (t * t).sum(-1)) if squared else (t.sum(-1), t.abs().sum(-1))
    k = chain + 4
    dI = (k * U + ep) * AI + 2.0 ** -40 * AI
    dP = (k * U + (2 * ep if squared else ep)) * AP + 2.0 ** -40 * AP
    dT = (k * U * AT if soft_target else 0.0 * AT) + 2.0 ** -40 * AT
    if batch:
        I, P, T, dI, dP, dT = (v.sum(0, keepdim=True) for v in (I, P, T, dI, dP, dT))
    D, dD = P + T, dP + dT
    if jaccard:
        D, dD = 2 * (D - I), 2 * (dD + dI)
    Dd, num, dnum = D + dr, 2 * I + nr, 2 * dI
    f = 1 - num / Dd
    df = dnum / Dd + num.abs() * dD / Dd ** 2
    terms = (1 if batch else N) * (C - c_lo)
    w = lambda_dice * (1.0 / terms if reduction == "mean" else 1.0)
    dice, ddice = w * f[:, c_lo:].sum(), w * df[:, c_lo:].sum()
    if jaccard:
        dFdI = -2 / Dd - 2 * num / Dd ** 2
        dFdP = 2 * num / Dd ** 2
        edI = 2 * dD / Dd ** 2 + 2 * dnum / Dd ** 2 + 4 * num.abs() * dD / Dd ** 3
        edP = 2 * (dnum / Dd ** 2 + 2 * num.abs() * dD / Dd ** 3)
    else:
        dFdI, dFdP = -2 / Dd, num / Dd ** 2
        edI, edP = 2 * dD / Dd ** 2, dnum / Dd ** 2 + 2 * num.abs() * dD / Dd ** 3
    keep = torch.ones(C, dtype=f64, device=x.device)
    keep[:c_lo] = 0
    a, b = (w * go * dFdI * keep).expand(N, C)[..., None], (w * go * dFdP * keep).expand(N, C)[..., None]
    da = (abs(w * go) * edI * keep).expand(N, C)[..., None] + U * a.abs()
    db = (abs(w * go) * edP * keep).expand(N, C)[..., None] + U * b.abs()
    # cross-entropy on the raw logits, summed per voxel in fp64
    ce_scale = lambda_ce * (1.0 / (N * S) if reduction == "mean" else 1.0)
    ep_ce = act_error("sigmoid" if C == 1 else "softmax", C, X)
    if C == 1:
        qce = torch.sigmoid(x)
        ce_v = x.clamp_min(0) - x * t + torch.log1p(torch.exp(-x.abs()))
        ace = x.abs() + (x * t).abs() + 1
        ce_grad_core = qce - t
        ce_grad_abs = qce + t.abs()
    else:
        qce = torch.softmax(x, 1)
        tsum = t.sum(1, keepdim=True)
        lse = torch.logsumexp(x, 1, keepdim=True)
        ce_v = lse * tsum - (t * x).sum(1, keepdim=True)
        ace = (lse.abs() + 1) * tsum.abs() + (t * x).abs().sum(1, keepdim=True)
        ce_grad_core = qce * tsum - t
        ce_grad_abs = qce * tsum.abs() + t.abs()
    ce, dce = ce_scale * ce_v.sum(), ce_scale * (C + 8 + 4.5 * X) * U * ace.sum()
    loss = dice + (ce if with_ce else 0.0)
    dloss = ddice + (dce if with_ce else 0.0) + U * abs(float(loss)) + 2.0 ** -40 * (abs(float(dice)) + abs(float(ce)))
    # dlogits: the fp32 evaluation of the kernel's expression from the (perturbed) coefficients
    g = a * t + b * q
    dq = 2 * p * ep if squared else 0.0
    dg = da * t.abs() + db * q.abs() + b.abs() * dq + 2 * U * ((a * t).abs() + (b * q).abs())
    if act == "softmax":
        s = (p * g).sum(1, keepdim=True)
        ds = (ep * p * g.abs() + p * dg).sum(1, keepdim=True) + (C + 1) * U * (p * g.abs()).sum(1, keepdim=True)
        dgrad = p * (g - s)
        ddg = ep * p * (g - s).abs() + p * (dg + ds) + 2 * U * p * (g.abs() + s.abs())
    elif act == "sigmoid":
        dp = p * (1 - p)
        dgrad = g * dp
        ddg = dg * dp + g.abs() * (2 * ep + 3 * U) * p + U * (g * dp).abs()
    else:
        dgrad, ddg = g, dg
    dx, ddx = dgrad, ddg
    if with_ce:
        cg = ce_scale * go
        dx = dx + cg * ce_grad_core
        ddx = ddx + abs(cg) * (ep_ce * qce * (1 if C == 1 else tsum.abs()) + 3 * U * ce_grad_abs)
    ddx = (ddx + U * dx.abs()) * (1 + 1e-6)
    return float(loss), float(dloss) * (1 + 1e-6), dx, ddx


def autograd_reference(x, t, *, act, squared, jaccard, batch, include_background, reduction, lambda_dice=1.0, lambda_ce=0.0,
                       with_ce=False, go, nr=1e-5, dr=1e-5, **_):
    """the same loss through fp64 autograd, term by term as MONAI writes it (checks the closed forms above)"""
    x = x.clone().requires_grad_(True)
    N, C, S = x.shape
    p = torch.sigmoid(x) if act == "sigmoid" else torch.softmax(x, 1) if act == "softmax" else x
    pp, tt = (p[:, 1:], t[:, 1:]) if (not include_background and C > 1) else (p, t)
    axes = [0, 2] if batch else [2]
    inter = (pp * tt).sum(axes)
    den = ((pp * pp).sum(axes) + (tt * tt).sum(axes)) if squared else (pp.sum(axes) + tt.sum(axes))
    if jaccard:
        den = 2 * (den - inter)
    f = 1 - (2 * inter + f32(nr)) / (den + f32(dr))
    loss = f32(lambda_dice) * (f.mean() if reduction == "mean" else f.sum())
    if with_ce:
        if C == 1:
            ce = F.binary_cross_entropy_with_logits(x, t, reduction="sum")
        else:
            ce = -(t * torch.log_softmax(x, 1)).sum()
        loss = loss + f32(lambda_ce) * (ce / (N * S) if reduction == "mean" else ce)
    (dx,) = torch.autograd.grad(loss, x, torch.tensor(go, dtype=f64, device=x.device))
    return float(loss.detach()), dx


def check_against_autograd(x, t, kw, loss, dx):
    al, adx = autograd_reference(x, t, **kw)
    assert abs(al - loss) <= 1e-12 * max(1.0, abs(al))
    assert float((adx - dx).abs().max()) <= 1e-12 * max(1e-30, float(adx.abs().max()))


def flag_sets(n_logits, names):
    """every combination of the boolean flags, or four that between them set each flag both ways"""
    full = [dict(zip(names, bits)) for bits in itertools.product((False, True), repeat=len(names))]
    if n_logits <= FULL_PRODUCT_MAX:
        return full
    pick = [(0,) * len(names), (1,) * len(names), tuple(i % 2 for i in range(len(names))), tuple((i + 1) % 2 for i in range(len(names)))]
    return [dict(zip(names, map(bool, bits))) for bits in pick]


# ---------------------------------------------------------------------------------------------------------------- Dice
def _misaligned(v, dtype):
    """v as a contiguous view one element into a larger buffer"""
    buf = torch.zeros(v.numel() + 1, dtype=dtype, device=DEV)
    buf[1:] = v.flatten()
    return buf[1:].view(v.shape)


@pytest.mark.parametrize("case", B.DICE_CASES, ids=lambda c: c.id)
def test_dice_loss_and_dlogits_match_fp64(pkg, case):
    n, c, S, target = case.args[:4]
    aligned = case.args[4] if len(case.args) > 4 else True
    geo = B.dice_geometry(n, c, S, target, aligned)
    gen = gen_of(case.id)
    x_sig = torch.randn(n, c, S, generator=gen, device=DEV) * 2.5
    x_id = torch.rand(n, c, S, generator=gen, device=DEV)            # sigmoid=False: the logits are the probabilities
    if target == "u8":
        tt = (torch.rand(n, c, S, generator=gen, device=DEV) > 0.7).to(torch.uint8)
    else:
        tt = torch.rand(n, c, S, generator=gen, device=DEV)
    mis = case.opt.get("misaligned")
    t_in = _misaligned(tt, tt.dtype) if mis == "target" else tt
    if mis:
        assert (t_in.data_ptr() % 4 != 0) if mis == "target" else True
    t64 = tt.double()
    names = ("sigmoid", "squared_pred", "jaccard", "batch", "include_background", "sum")
    for i, fl in enumerate(flag_sets(n * c * S, names)):
        go = f32(GRAD_OUTS[i % len(GRAD_OUTS)])
        x = x_sig if fl["sigmoid"] else x_id
        x_in = _misaligned(x, torch.float32) if mis == "logits" else x
        if mis == "logits":
            assert x_in.data_ptr() % 16 != 0
        xq = x_in.detach().requires_grad_(True)
        kw = dict(sigmoid=fl["sigmoid"], squared_pred=fl["squared_pred"], jaccard=fl["jaccard"], batch=fl["batch"],
                  include_background=fl["include_background"], reduction="sum" if fl["sum"] else "mean")
        loss = pkg.DiceLoss(**kw)(xq, t_in)
        (dx,) = torch.autograd.grad(loss, xq, torch.tensor(go, device=DEV))
        rkw = dict(act="sigmoid" if fl["sigmoid"] else None, squared=kw["squared_pred"], jaccard=kw["jaccard"], batch=kw["batch"],
                   include_background=kw["include_background"], reduction=kw["reduction"], go=go)
        x64 = x.double()
        ref, lim, rdx, dlim = reference(x64, t64, chain=geo["chain"], soft_target=target == "f32", **rkw)
        if n * c * S <= 1 << 16:
            check_against_autograd(x64, t64, rkw, ref, rdx)
        what = "%s %s grad_out %g" % (case.id, kw, go)
        err = abs(float(loss.detach()) - ref)
        assert err <= lim, "%s: loss %.10g ref %.10g bound %.3g" % (what, float(loss.detach()), ref, lim)
        note(case, "loss", err / lim)
        note(case, "dlogits", within(dx, rdx, dlim, what + " dlogits"))
        # the C2-size rows hold 537 M logits: free this flag set's fp64 tensors (4.3 GB each) before the next one's
        del loss, dx, rdx, dlim, x64, xq


# ------------------------------------------------------------------------------------------------------ Dice + CE
def dice_ce_targets(case, gen):
    """(target as DiceCELoss takes it, the [N, C, S] fp64 target the kernels see)"""
    n, c, S, kind = case.args[:4]
    if kind == "soft_f32":
        t = torch.rand(n, c, S, generator=gen, device=DEV)
        return t, t.double()
    if c == 1:
        t = (torch.rand(n, 1, S, generator=gen, device=DEV) > 0.6).to(torch.uint8)
        return t, t.double()
    lab = torch.randint(0, c, (n, 1, S), generator=gen, device=DEV)
    out = torch.rand(n, 1, S, generator=gen, device=DEV) < 0.03    # labels outside [0, C): all-zero target rows
    valid = (~out).double()
    onehot = F.one_hot(lab[:, 0], c).permute(0, 2, 1).double() * valid
    if kind == "label_u8":
        return lab.masked_fill(out, 255).to(torch.uint8), onehot
    if kind == "label_i64":
        return lab.masked_fill(out, -1).masked_fill(out & (torch.rand(n, 1, S, generator=gen, device=DEV) < 0.5), c), onehot
    return onehot.to(torch.uint8), onehot


@pytest.mark.parametrize("case", B.DICE_CE_CASES, ids=lambda c: c.id)
def test_dice_ce_loss_and_dlogits_match_fp64(pkg, case):
    n, c, S, kind, act, with_ce = case.args
    geo = B.dice_ce_geometry(n, c, S, kind, act)
    gen = gen_of(case.id)
    x = torch.rand(n, c, S, generator=gen, device=DEV) if geo["act"] is None else torch.randn(n, c, S, generator=gen, device=DEV) * 2.5
    t_in, t64 = dice_ce_targets(case, gen)
    label_map = kind.startswith("label") and c > 1
    x64 = x.double()
    names = ("squared_pred", "jaccard", "batch", "include_background", "sum")
    for i, fl in enumerate(flag_sets(n * c * S, names)):
        go = f32(GRAD_OUTS[i % len(GRAD_OUTS)])
        lam_d, lam_ce = (1.0, 1.0) if i % 2 == 0 else (0.6, 0.75)
        if not with_ce:
            lam_ce = 0.0
        kw = dict(softmax=act == "softmax", sigmoid=act == "sigmoid", to_onehot_y=label_map, squared_pred=fl["squared_pred"],
                  jaccard=fl["jaccard"], batch=fl["batch"], include_background=fl["include_background"],
                  reduction="sum" if fl["sum"] else "mean", lambda_dice=lam_d, lambda_ce=lam_ce)
        xq = x.clone().requires_grad_(True)
        loss = pkg.DiceCELoss(**kw)(xq.view(n, c, S, 1, 1), t_in.view(t_in.shape[0], t_in.shape[1], S, 1, 1))
        (dx,) = torch.autograd.grad(loss, xq, torch.tensor(go, device=DEV))
        rkw = dict(act=geo["act"], squared=kw["squared_pred"], jaccard=kw["jaccard"], batch=kw["batch"],
                   include_background=kw["include_background"], reduction=kw["reduction"], lambda_dice=lam_d, lambda_ce=lam_ce,
                   with_ce=with_ce, go=go)
        ref, lim, rdx, dlim = reference(x64, t64, chain=geo["chain"], soft_target=kind == "soft_f32", **rkw)
        if n * c * S <= 1 << 16:
            check_against_autograd(x64, t64, rkw, ref, rdx)
        what = "%s %s grad_out %g" % (case.id, kw, go)
        err = abs(float(loss.detach()) - ref)
        assert err <= lim, "%s: loss %.10g ref %.10g bound %.3g" % (what, float(loss.detach()), ref, lim)
        note(case, "loss", err / lim)
        note(case, "dlogits", within(dx, rdx, dlim, what + " dlogits"))


# ---------------------------------------------------------------------------------------------------------- tiling
class TileNet:
    """a network whose output depends on the tile-local position and mixes channels (cin -> cout), evaluated in fp64 and
    rounded once to fp32 when called by the inferer"""

    def __init__(self, cin, cout, roi, gen):
        self.w = torch.randn(cout, cin, generator=gen, device=DEV).double()
        self.b = torch.randn(cout, generator=gen, device=DEV).double()
        z, y, x = torch.meshgrid(*[torch.arange(r, device=DEV, dtype=f64) / r for r in roi], indexing="ij")
        self.ramp = torch.stack([(o + 1) * 0.5 * z - 0.3 * y + 0.2 * (o % 3) * x for o in range(cout)])

    def f64(self, tiles):
        return torch.einsum("oc,bcdhw->bodhw", self.w, tiles) + self.b.view(1, -1, 1, 1, 1) + self.ramp

    def __call__(self, tiles):
        return self.f64(tiles.double()).float()


@pytest.mark.parametrize("case", B.TILE_CASES, ids=lambda c: c.id)
def test_tiling_kernels_match_fp64_weighted_average(pkg, case):
    shape, roi, overlap, swb, cout = case.args
    geo = B.tiling_geometry(*case.args)
    n, cin, D, H, W = shape
    gen = gen_of(case.id)
    x = torch.randn(shape, generator=gen, device=DEV) + 4.0 * torch.arange(n, device=DEV).view(n, 1, 1, 1, 1)   # samples differ
    r = geo["roi"]
    net = TileNet(cin, cout, r, gen)
    _, _, jobs, _ = B.tiling_plan(shape, roi, overlap, swb)
    for mode in ("constant", "gaussian"):
        inf = pkg.predict.SlidingWindowInferer(roi_size=roi, sw_batch_size=swb, overlap=overlap, mode=mode)
        with torch.no_grad():
            got = inf(x, net)
            again = inf(x, net)
        assert torch.equal(got, again), "%s %s: not bit-identical when run again" % (case.id, mode)
        r_used, imp, axes, _ = inf._scan((D, H, W), x.device)
        assert tuple(r_used) == r and axes == geo["axes"]
        imp64 = imp.double()                     # the importance map the kernels read, fp32
        acc = torch.zeros(n, cout, D, H, W, dtype=f64, device=DEV)
        aabs = torch.zeros_like(acc)
        wsum = torch.zeros(D, H, W, dtype=f64, device=DEV)
        cover = torch.zeros(D, H, W, dtype=f64, device=DEV)
        for b, d, h, w in jobs:
            box = (slice(d, d + r[0]), slice(h, h + r[1]), slice(w, w + r[2]))
            pred = net(x[b:b + 1, :, box[0], box[1], box[2]]).double()[0]       # the fp32 tile prediction the kernels see
            acc[(b, slice(None)) + box] += pred * imp64
            aabs[(b, slice(None)) + box] += pred.abs() * imp64
            if b == 0:
                wsum[box] += imp64
                cover[box] += 1
        ref = acc / wsum
        # scatter: a chain of k products and sums per voxel; count: k fp32 additions; one division
        lim = U * (2 * cover * aabs / wsum + (cover + 2) * ref.abs()) * 1.01
        note(case, mode, within(got, ref, lim, "%s %s" % (case.id, mode)))
        assert int(cover.max()) == geo["max_cover"]


# ---------------------------------------------------------------------------------------------------------- z-score
def zscore_input(case, gen):
    c, dims, nonzero, _ = case.args
    x = torch.randn(c, *dims, generator=gen, device=DEV)
    x[0] = x[0] * 1.5 + 3000.0                                   # mean / std = 2000
    x[1] = 0.0                                                   # all zero
    x[2] = 7.25                                                  # constant
    x[3] = x[3] * 5 + 3
    x[3][torch.rand(dims, generator=gen, device=DEV) < 0.3] = 0.0   # background voxels
    return x


@pytest.mark.parametrize("case", B.ZSCORE_CASES, ids=lambda c: c.id)
def test_zscore_matches_fp64(pkg, case):
    c, dims, nonzero, channel_wise = case.args
    gen = gen_of(case.id)
    x = zscore_input(case, gen)
    got = pkg.prepost.normalize_intensity(x, nonzero=nonzero, channel_wise=channel_wise)
    groups = c if channel_wise else 1
    S = x.numel() // groups
    sweeps = B.zscore_geometry(groups, S)["sweeps"]
    xg, gg = x.double().reshape(groups, S), got.reshape(groups, S)
    sel = (xg != 0) if nonzero else torch.ones_like(xg, dtype=torch.bool)
    cnt = sel.sum(1, keepdim=True).double()
    xs = torch.where(sel, xg, torch.zeros_like(xg))
    mean = torch.where(cnt > 0, xs.sum(1, keepdim=True) / cnt.clamp_min(1), torch.zeros_like(cnt))
    var = torch.where(cnt > 0, (torch.where(sel, xg - mean, torch.zeros_like(xg)) ** 2).sum(1, keepdim=True) / cnt.clamp_min(1),
                      torch.zeros_like(cnt))
    sd = var.sqrt()
    ex2 = torch.where(cnt > 0, (xs ** 2).sum(1, keepdim=True) / cnt.clamp_min(1), torch.zeros_like(cnt))
    # the kernel's fp64 statistics: per-thread chains of `sweeps` terms, a block tree and one atomic add per chunk; var = E[x^2] - mean^2
    e64 = (sweeps + 16 + B.zscore_geometry(groups, S)["chunks"]) * U64
    dmean = e64 * xs.abs().sum(1, keepdim=True) / cnt.clamp_min(1)
    dvar = 3 * e64 * ex2 + 2 * mean.abs() * dmean
    zero_sd = sd == 0
    sd = torch.where(zero_sd, torch.ones_like(sd), sd)
    rel_sd = torch.where(zero_sd, torch.zeros_like(sd), dvar / (2 * var.clamp_min(1e-300)))
    assert bool((rel_sd < 1e-3).all()), "the statistics are too ill-conditioned for the model"
    ref = torch.where(sel, (xg - mean) / sd, xg)
    # (x - (float)mean) * (float)(1 / sd): the fp32 mean is off by |mean| u; subtraction, reciprocal and product round once each
    lim = (mean.abs() * U + dmean) / sd + ref.abs() * (3 * U + rel_sd)
    lim = torch.where(sel, lim * 1.01, torch.zeros_like(lim))   # unselected voxels are copied exactly
    note(case, "y", within(gg, ref, lim, case.id))
    if nonzero:
        assert bool((gg[~sel] == 0).all())
    if channel_wise:
        assert bool((gg[1] == 0).all()) and bool((gg[2] == 0).all())   # all-zero and constant channels: 0 after normalising
