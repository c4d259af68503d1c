"""Every kernel route of the convolution and the weight gradient (tests/conv_route_cases.py) against an fp64 reference, element by
element.  Each case first checks through the host query that it still takes its route, then launches it on inputs the
reference reads exactly (bf16 hi, or hi + lo, as stored), and bounds every element by

    |got - ref| <= r * |ref| + a * (|x| conv |w|)

with r the rounding of the stored precision (2^-8 bf16, 2^-16 hi + lo) and a the fp32 accumulation of the tensor cores; the
per-channel statistics of the fused epilogue are checked the same way against the values before the bf16 rounding.  The
plan-only options (bias, zeroed boundary, visible extents, deterministic weight-gradient partial sums) run through the
diagnostics entry points of include/b200unet_diag.h."""
import zlib

import pytest
import torch
import torch.nn.functional as F

import conv_route_cases as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
R_STORE = {False: 2.0 ** -8, True: 2.0 ** -16}    # rounding of a stored bf16 / hi + lo value
A_ACC = 2.0 ** -15                                # fp32 accumulation, relative to sum |x| |w|
SENTINEL = 7.0
C0 = 8                                            # the output view starts at channel 8 of a wider buffer
G = 8                                             # GroupNorm groups of the mode-1 cases


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


# -------------------------------------------------------------------------------------------------------------- helpers
def make_act(L, v, c_view, split):
    """fp32 NCDHW values v -> Act with c_view channels (the rest zero) and the exact fp64 NCDHW value it stores"""
    n, c, d, h, w = v.shape
    full = torch.zeros(n, d, h, w, c_view, device=DEV)
    full[..., :c] = v.permute(0, 2, 3, 4, 1).to(DEV)
    hi = full.bfloat16()
    lo = (full - hi.float()).bfloat16() if split else None
    act = L.Act(hi.contiguous(), lo.contiguous() if split else None)
    val = hi.double() + (lo.double() if split else 0)
    return act, val.permute(0, 4, 1, 2, 3)[:, :c].cpu()


def rand_act(L, n, c, dims, split, gen, c_view=None, shift=0.0):
    v = torch.randn(n, c, *dims, generator=gen) + shift
    return make_act(L, v, c_view or c, split)


def packed(L, w, mode, split, cop=None):
    """pack w; returns (hi, lo, exact fp64 value of the pack in w's own layout)"""
    hi, lo, cop_, cip, T = L.pack_weights(w.to(DEV), mode, split=split, cop=cop)
    q = (hi.double() + (lo.double() if split else 0)).cpu()
    if mode == 0:      # [T][Cop][Cip] <- [Co][Ci][k^3]
        co, ci = w.shape[:2]
        wq = q[:, :co, :ci].permute(1, 2, 0).reshape(w.shape)
    elif mode == 4:    # [T][Cop][Cip] <- ConvTranspose3d [Ci][Co][k^3]
        ci, co = w.shape[:2]
        wq = q[:, :co, :ci].permute(2, 1, 0).reshape(w.shape)
    else:
        raise ValueError(mode)
    return hi, lo, wq


def check_elements(got, ref, bound_abs, r, what, mask=None):
    """|got - ref| <= r |ref| + bound_abs at every element (of mask); the message names the worst element"""
    err = (got - ref).abs()
    lim = r * ref.abs() + bound_abs + 1e-30
    bad = err > lim
    if mask is not None:
        bad &= mask
    if bool(bad.any()):
        idx = tuple(int(i) for i in (bad.nonzero()[0]))
        pytest.fail("%s: %d of %d elements out of bounds; first at %s (n, c, d, h, w): got %.8g ref %.8g bound %.3g"
                    % (what, int(bad.sum()), bad.numel(), idx, float(got[idx]), float(ref[idx]), float(lim[idx])))


def view_value(act):
    """exact fp64 NCDHW value of an Act's visible channels"""
    v = act.hi[..., act.c0:act.c0 + act.c].double()
    if act.lo is not None:
        v = v + act.lo[..., act.c0:act.c0 + act.c].double()
    return v.permute(0, 4, 1, 2, 3).cpu()


def assert_route(r, case):
    assert (r["kind"], r["bn"], r["kc"], r["kchunks"]) == (case.kind, case.bn, case.kc, case.kchunks), r


# ----------------------------------------------------------------------------------------------------------- convolution
def conv_inputs(L, case, gen, real_out):
    """sources, packed weights and the fp64 forward pieces of a case: returns (call args, call kwargs, acc, absacc)"""
    n = 2
    sdims, ksz, stride, cls = R.conv_geometry(case.op, case.cin, case.dims)
    x, xv = rand_act(L, n, case.cin, sdims, case.split, gen)
    if cls == 1:       # data gradient of a k3 s2 p1 convolution real_out -> cin: the mode-1 pack of its weight
        w = torch.randn(case.cin, real_out, 3, 3, 3, generator=gen) / (case.cin * 27) ** 0.5
        whi, wlo, _, _, _ = L.pack_weights(w.to(DEV), 1, split=case.split, cip=case.cout)
        _, _, wq = packed(L, w, 0, case.split, cop=None)
        acc = F.conv_transpose3d(xv, wq, stride=2, padding=1, output_padding=1)
        absacc = F.conv_transpose3d(xv.abs(), wq.abs(), stride=2, padding=1, output_padding=1)
    elif cls == 2:     # ConvTranspose3d(cin -> real_out, kernel = stride = 2): the mode-4 pack
        w = torch.randn(case.cin, real_out, 2, 2, 2, generator=gen) / case.cin ** 0.5
        whi, wlo, wq = packed(L, w, 4, case.split, cop=case.cout)
        acc = F.conv_transpose3d(xv, wq, stride=2)
        absacc = F.conv_transpose3d(xv.abs(), wq.abs(), stride=2)
    else:
        w = torch.randn(real_out, case.cin, ksz, ksz, ksz, generator=gen) / (case.cin * ksz ** 3) ** 0.5
        whi, wlo, wq = packed(L, w, 0, case.split, cop=case.cout)
        acc = F.conv3d(xv, wq, stride=stride, padding=ksz // 2)
        absacc = F.conv3d(xv.abs(), wq.abs(), stride=stride, padding=ksz // 2)
    kw = dict(cls_mode=cls)
    if case.cin2:
        x2, x2v = rand_act(L, n, case.cin2, case.dims, case.split, gen)
        w2 = torch.randn(real_out, case.cin2, 1, 1, 1, generator=gen) / case.cin2 ** 0.5
        w2hi, w2lo, w2q = packed(L, w2, 0, case.split, cop=case.cout)
        acc = acc + F.conv3d(x2v, w2q)
        absacc = absacc + F.conv3d(x2v.abs(), w2q.abs())
        kw.update(x2=x2, w2_hi=w2hi, w2_lo=w2lo, cip2=case.cin2)
    return (x, whi, wlo, ksz, stride), kw, acc, absacc


def wide_out(L, n, dims, cout, split):
    """a buffer of C0 + cout + 8 channels filled with the sentinel; the case writes the view [C0, C0 + cout)"""
    buf = L.Act.empty(n, *dims, C0 + cout + 8, split=split)
    buf.hi.fill_(SENTINEL)
    if split:
        buf.lo.fill_(SENTINEL / 256)
    return buf


def check_untouched(buf, cout, split):
    for t in ([buf.hi, buf.lo] if split else [buf.hi]):
        outside = torch.cat([t[..., :C0], t[..., C0 + cout:]], dim=-1)
        assert bool((outside == outside.flatten()[0]).all()) and float(outside.flatten()[0]) != 0.0, "write outside the view"


def run_mode0(L, case, gen, ext=None, edit_ref=None):
    """(acc + residual) * dropout scale [+ bias] -> the view at C0 of a sentinel-filled buffer, with the statistics"""
    n = 2
    real_out = case.cout - 4                     # the last 4 channels of the view are weight padding: stored as exact zeros
    args, kw, acc, absacc = conv_inputs(L, case, gen, real_out)
    res, resv = rand_act(L, n, real_out, case.dims, case.split, gen, c_view=case.cout)
    scale = torch.tensor([0.0, 0.8, 1.25])[torch.randint(0, 3, (n, case.cout), generator=gen)].to(DEV)
    buf = wide_out(L, n, case.dims, case.cout, case.split)
    out = buf.slice(C0, case.cout)
    stats = torch.zeros(n, C0 + case.cout + 8, 2, dtype=torch.float64, device=DEV)
    kw.update(res=res, scale=scale, stats=stats[:, C0:], stats_ld=C0 + case.cout + 8)
    x, whi, wlo, ksz, stride = args
    route = R.with_wide_env(case.wide, lambda: L.conv3d_route(x, whi, wlo, ksz, stride, out, case.cout, case.cin, ext=ext, **kw))
    assert_route(route, case)
    R.with_wide_env(case.wide, lambda: L.conv3d_ex(x, whi, wlo, ksz, stride, out, case.cout, case.cin, ext=ext, **kw))
    torch.cuda.synchronize()
    s = scale.double().cpu()[:, :real_out, None, None, None]
    ref = (acc + resv) * s
    bound = A_ACC * absacc * s
    if edit_ref is not None:
        ref, bound = edit_ref(ref, bound)
    got = view_value(out)
    check_elements(got[:, :real_out], ref, bound, R_STORE[case.split], "output")
    assert float(got[:, real_out:].abs().max()) == 0.0, "padded output channels"
    check_untouched(buf, case.cout, case.split)
    # statistics of the values before the bf16 rounding
    st = stats.cpu()
    assert float(st[:, :C0].abs().max()) == 0.0 and float(st[:, C0 + case.cout:].abs().max()) == 0.0
    sm = st[:, C0:C0 + real_out]
    dims = (2, 3, 4)
    b1 = bound.sum(dim=dims) + 2.0 ** -16 * ref.abs().sum(dim=dims) + 1e-9
    b2 = (2 * ref.abs() * bound + bound * bound).sum(dim=dims) + 2.0 ** -16 * (ref * ref).sum(dim=dims) + 1e-9
    assert bool(((sm[..., 0] - ref.sum(dim=dims)).abs() <= b1).all()), "per-channel sums"
    assert bool(((sm[..., 1] - (ref * ref).sum(dim=dims)).abs() <= b2).all()), "per-channel sums of squares"
    assert float(st[:, C0 + real_out:C0 + case.cout].abs().max()) == 0.0
    return route


def run_mode1(L, case, gen, slope):
    """GroupNorm/activation backward epilogue: dz = acc * act'(A x + B), (sum dz, sum dz * xhat) per channel"""
    n = 2
    args, kw, acc, absacc = conv_inputs(L, case, gen, case.cout)
    gx, gxv = rand_act(L, n, case.cout, case.dims, case.split, gen, shift=0.3)
    gamma = (torch.randn(case.cout, generator=gen) * 0.3 + 1).to(DEV)
    beta = (torch.randn(case.cout, generator=gen) * 0.2).to(DEV)
    v = gxv
    st_in = torch.stack([v.sum(dim=(2, 3, 4)), (v * v).sum(dim=(2, 3, 4))], dim=-1).contiguous().to(DEV)
    coef = torch.empty(n, case.cout, 4, device=DEV)
    L.gn_apply(gx, L.Act.empty(n, *case.dims, case.cout, split=case.split), st_in, gamma, beta, case.cout, G, coef, slope=slope)
    bst = torch.zeros(n, case.cout, 2, dtype=torch.float64, device=DEV)
    dz = L.Act.empty(n, *case.dims, case.cout, split=case.split)
    dz.hi.fill_(SENTINEL)
    kw.update(mode=1, gn_x=gx, coef=coef, coef_ld=case.cout, slope=slope, bstats=bst)
    x, whi, wlo, ksz, stride = args
    route = R.with_wide_env(case.wide, lambda: L.conv3d_route(x, whi, wlo, ksz, stride, dz, case.cout, case.cin, **kw))
    assert_route(route, case)
    R.with_wide_env(case.wide, lambda: L.conv3d(x, whi, wlo, ksz, stride, dz, case.cout, case.cin, **kw))
    torch.cuda.synchronize()
    xq = gxv.clone().requires_grad_(True)
    z = F.group_norm(xq, G, gamma.double().cpu(), beta.double().cpu(), 1e-5)
    z.retain_grad()
    F.leaky_relu(z, slope).backward(acc)
    ref = z.grad
    bound = A_ACC * absacc
    clear = z.detach().abs() > 1e-3          # the fp32 A x + B of the kernel decides the sign of these exactly as fp64 does
    got = view_value(dz)
    check_elements(got, ref, bound, R_STORE[case.split], "dz (slope %g)" % slope, mask=clear)
    mu, rstd = coef[..., 2].double().cpu(), coef[..., 3].double().cpu()
    xhat = (gxv - mu[:, :, None, None, None]) * rstd[:, :, None, None, None]
    dims = (2, 3, 4)
    amb = (~clear).double() * acc.abs()       # an undecided sign moves that element's dz by at most |acc|
    b1 = bound.sum(dim=dims) + amb.sum(dim=dims) + 2.0 ** -16 * ref.abs().sum(dim=dims) + 1e-9
    b2 = ((bound + amb) * xhat.abs()).sum(dim=dims) + 2.0 ** -16 * (ref * xhat).abs().sum(dim=dims) + 1e-9
    b = bst.cpu()
    assert bool(((b[..., 0] - ref.sum(dim=dims)).abs() <= b1).all()), "sum dz (slope %g)" % slope
    assert bool(((b[..., 1] - (ref * xhat).sum(dim=dims)).abs() <= b2).all()), "sum dz * xhat (slope %g)" % slope


@pytest.mark.parametrize("case", R.CONV_CASES, ids=lambda c: c.id)
def test_conv_route_matches_fp64(L, case):
    gen = torch.Generator().manual_seed(zlib.crc32(case.id.encode()))
    if case.mode == 0:
        run_mode0(L, case, gen)
    else:
        for slope in (0.0, 0.01):
            run_mode1(L, case, gen, slope)


# -------------------------------------------------------------------------------------------------- plan-only conv options
PLAN_CASES = [R.ConvCase("halo", 32, 32, False, 0, 1, "k3s1", 32, 24, R.H), R.ConvCase("tap", 32, 32, False, 0, 1, "k3s1", 32, 24, R.P),
              R.ConvCase("tap", 32, 32, True, 0, 1, "k3s1", 32, 24, R.P), R.ConvCase("tap", 64, 64, False, 0, 1, "k3s1", 64, 40, R.P)]


@pytest.mark.parametrize("case", PLAN_CASES, ids=lambda c: c.id)
def test_conv_bias_and_zeroed_boundary(L, case):
    """the transposed-convolution epilogue of the plans: + bias, then the high boundary plane, row and column stored as 0; the
    statistics follow the stored zeros"""
    gen = torch.Generator().manual_seed(11)
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
    run_mode0(L, case, gen, ext=L.diag_ext(bias=bias, zero_last=True), edit_ref=edit)


@pytest.mark.parametrize("case", PLAN_CASES[:3], ids=lambda c: c.id)
def test_conv_visible_extents_one_short(L, case):
    """a source whose last plane, row and column lie beyond its visible extents reads them as zero (the masked gradient of a
    padded transposed convolution)"""
    n = 2
    gen = torch.Generator().manual_seed(12)
    x, xv = rand_act(L, n, case.cin, case.dims, case.split, gen)
    w = torch.randn(case.cout, case.cin, 3, 3, 3, generator=gen) / (case.cin * 27) ** 0.5
    whi, wlo, wq = packed(L, w, 0, case.split)
    xz = xv.clone()
    xz[:, :, -1] = 0
    xz[:, :, :, -1] = 0
    xz[..., -1] = 0
    ext = L.diag_ext(x_vis=[tuple(v - 1 for v in case.dims)])
    y = L.Act.empty(n, *case.dims, case.cout, split=case.split)
    assert_route(L.conv3d_route(x, whi, wlo, 3, 1, y, case.cout, case.cin, ext=ext), case)
    L.conv3d_ex(x, whi, wlo, 3, 1, y, case.cout, case.cin, ext=ext)
    torch.cuda.synchronize()
    ref = F.conv3d(xz, wq, padding=1)
    check_elements(view_value(y), ref, A_ACC * F.conv3d(xz.abs(), wq.abs(), padding=1), R_STORE[case.split], "output")


# ------------------------------------------------------------------------------------------------------- weight gradient
def wgrad_inputs(L, case, gen, dy_vis=None):
    n = 2
    adims, ksz, stride = R.wgrad_geometry(case.op, case.dims)
    a, av = rand_act(L, n, case.ci, adims, case.split, gen)
    dy, dyv = rand_act(L, n, case.co, case.dims, case.split, gen)
    if dy_vis:
        dyv = dyv.clone()
        dyv[:, :, dy_vis[0]:] = 0
        dyv[:, :, :, dy_vis[1]:] = 0
        dyv[..., dy_vis[2]:] = 0
    pad = 0 if ksz == 2 else ksz // 2
    wz = torch.zeros(case.co, case.ci, ksz, ksz, ksz, dtype=torch.float64, requires_grad=True)
    F.conv3d(av, wz, stride=stride, padding=pad).backward(dyv)
    ref = wz.grad.permute(2, 3, 4, 1, 0).reshape(ksz ** 3, case.ci, case.co)
    wz.grad = None
    F.conv3d(av.abs(), wz, stride=stride, padding=pad).backward(dyv.abs())
    bound = A_ACC * wz.grad.permute(2, 3, 4, 1, 0).reshape(ksz ** 3, case.ci, case.co)
    return a, dy, ksz, stride, ref, bound


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("case", R.WGRAD_CASES, ids=lambda c: c.id)
def test_wgrad_route_matches_fp64(L, case):
    gen = torch.Generator().manual_seed(zlib.crc32(case.id.encode()))
    a, dy, ksz, stride, ref, bound = wgrad_inputs(L, case, gen)
    T, ci, co = ksz ** 3, case.ci, case.co
    r = L.wgrad_route(a, dy, ksz, stride, ci, co, num_sms=sms())
    assert R.wgrad_route_key(case.split, r) == case.key, r
    # atomic accumulation into a zeroed dw
    dw = torch.zeros(T, ci, co, device=DEV)
    assert L.wgrad_ex(a, dy, ksz, stride, ci, co, dw) == 0
    torch.cuda.synchronize()
    check_elements(dw.double().cpu(), ref, bound, 2.0 ** -20, "dw (atomics)")
    # deterministic partial sums + fixed-order reduction: the split count the route reports, bit-identical repeats
    rd = L.wgrad_route(a, dy, ksz, stride, ci, co, deterministic=True, num_sms=sms())
    assert rd["part_bytes"] == rd["splits"] * T * ci * co * 4
    plan_bytes = L.wgrad_partial_bytes(a, dy, ksz, stride, ci, co, num_sms=sms())
    assert plan_bytes >= rd["part_bytes"]
    part = torch.empty(plan_bytes // 4, device=DEV)
    outs = []
    for _ in range(2):
        dwd = torch.full((T, ci, co), float("nan"), device=DEV)
        assert L.wgrad_ex(a, dy, ksz, stride, ci, co, dwd, part=part) == rd["splits"]
        torch.cuda.synchronize()
        outs.append(dwd.clone())
    assert torch.equal(outs[0], outs[1]), "deterministic weight gradient differs between two runs"
    check_elements(outs[0].double().cpu(), ref, bound, 2.0 ** -20, "dw (deterministic)")
    # the partial buffer: exactly the route's bytes are enough, 4 bytes less is refused before any launch
    dwx = torch.zeros(T, ci, co, device=DEV)
    assert L.wgrad_ex(a, dy, ksz, stride, ci, co, dwx, part=part, part_bytes=rd["part_bytes"]) == rd["splits"]
    with pytest.raises(RuntimeError, match=r"status -1\).*partial buffer too small"):
        L.wgrad_ex(a, dy, ksz, stride, ci, co, dwx, part=part, part_bytes=rd["part_bytes"] - 4)
    torch.cuda.synchronize()
    assert torch.equal(dwx, outs[0])


@pytest.mark.parametrize("case", [c for c in R.WGRAD_CASES if c.kind == "halo"][:2] + [c for c in R.WGRAD_CASES if c.kind == "tap"][:3],
                         ids=lambda c: c.id)
def test_wgrad_dy_visible_extents_one_short(L, case):
    gen = torch.Generator().manual_seed(13)
    vis = tuple(v - 1 for v in case.dims)
    a, dy, ksz, stride, ref, bound = wgrad_inputs(L, case, gen, dy_vis=vis)
    ext = L.diag_ext(dy_vis=vis)
    assert R.wgrad_route_key(case.split, L.wgrad_route(a, dy, ksz, stride, case.ci, case.co, ext=ext, num_sms=sms())) == case.key
    dw = torch.zeros(ksz ** 3, case.ci, case.co, device=DEV)
    L.wgrad_ex(a, dy, ksz, stride, case.ci, case.co, dw, ext=ext)
    torch.cuda.synchronize()
    check_elements(dw.double().cpu(), ref, bound, 2.0 ** -20, "dw with dy visible one short")


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("c", [8, 40, 256])
def test_bias_grad_visible_extents_one_short(L, c, split):
    gen = torch.Generator().manual_seed(c)
    dims = (5, 6, 9)
    dy, dyv = rand_act(L, 2, c, dims, split, gen)
    db = torch.full((c,), float("nan"), device=DEV)
    L.bias_grad(dy, db, ext=L.diag_ext(dy_vis=(4, 5, 8)))
    torch.cuda.synchronize()
    z = dyv[:, :, :4, :5, :8]
    check_elements(db.double().cpu(), z.sum(dim=(0, 2, 3, 4)), 2.0 ** -16 * z.abs().sum(dim=(0, 2, 3, 4)), 0.0, "dbias")
