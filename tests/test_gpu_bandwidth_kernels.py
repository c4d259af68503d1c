"""The bandwidth-bound kernels of csrc/elementwise.cu against fp64, element by element, at the launch geometries the plans give
them (tests/bandwidth_cases.py): GroupNorm apply / backward / finalize, the activation backward, the x2 up-sampling forward and
backward, the fused up-sampling + skip-add, the transposed-convolution bias gradient and the 1..8-output head (forward, backward
and bias gradient), plus zero insertion, input packing, the input gradient and the layout converters.

Inputs are built in torch and rounded to bf16 there (hi, or hi + lo); the reference reads the exact fp64 value each one stores.
Outputs are read straight from their hi / lo tensors, never through the library's converters, and are views at channel 8 of
a sentinel-filled wider buffer: nothing outside the view may change.  Every element must satisfy

    |got - ref| <= r |ref| + a * ABS

with r the rounding of the stored result (2^-8 bf16, 2^-16 hi + lo), ABS the same expression evaluated on absolute values
and a the fp32 arithmetic of the kernel.  Values a kernel computes in fp64 and rounds once (GroupNorm coefficients, dgamma,
dbeta) are held to fp32 rounding; sums a thread accumulates in fp32 are held to the length of its chain, which the launch
geometry gives.  The fp64 references run on the device."""
import zlib

import pytest
import torch
import torch.nn.functional as F

import bandwidth_cases as B

pytestmark = pytest.mark.gpu

DEV = "cuda"
R_STORE = {False: 2.0 ** -8, True: 2.0 ** -16}
U = 2.0 ** -24                 # fp32 unit roundoff
SENTINEL = 7.0
C0 = 8                         # output views start at channel 8 of a wider buffer
f64 = torch.float64


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


def gen_of(name):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(name.encode()))


# -------------------------------------------------------------------------------------------------------------- helpers
def act_in(L, v, split, c_view=None, c0=0):
    """fp32 NDHWC values v [n, d, h, w, c] -> (Act view of c channels at c0 of a c_view-wide buffer, exact fp64 value [n, d, h, w, c])"""
    n, d, h, w, c = v.shape
    c_view = c_view or c0 + c
    full = torch.zeros(n, d, h, w, c_view, device=DEV)
    full[..., c0:c0 + c] = v
    hi = full.bfloat16()
    lo = (full - hi.float()).bfloat16() if split else None
    a = L.Act(hi.contiguous(), lo.contiguous() if split else None, c0, c)
    val = hi[..., c0:c0 + c].double() + (lo[..., c0:c0 + c].double() if split else 0)
    return a, val


def rand_in(L, n, c, dims, split, gen, scale=1.0, shift=0.0, c_view=None, c0=0):
    v = torch.randn(n, *dims, c, generator=gen, device=DEV) * scale + shift
    return act_in(L, v, split, c_view, c0)


def out_view(L, n, dims, c, split):
    """a buffer of C0 + c + 8 channels filled with the sentinel; returns (buffer, view at C0)"""
    buf = L.Act.empty(n, *dims, C0 + c + 8, split=split)
    buf.hi.fill_(SENTINEL)
    if split:
        buf.lo.fill_(SENTINEL / 256)
    return buf, buf.slice(C0, c)


def got_of(a):
    """exact fp64 value of a view, read from its hi / lo tensors"""
    v = a.hi[..., a.c0:a.c0 + a.c].double()
    return v + a.lo[..., a.c0:a.c0 + a.c].double() if a.lo is not None else v


def untouched(buf, c):
    for t in ([buf.hi, buf.lo] if buf.lo is not None else [buf.hi]):
        outside = torch.cat([t[..., :C0], t[..., C0 + c:]], dim=-1)
        first = outside.flatten()[0]
        assert float(first) != 0.0 and bool((outside == first).all()), "a write outside the output view"


def check(got, ref, absb, r, a, what, mask=None):
    """|got - ref| <= r |ref| + a * absb at every element (of mask); names the worst element.  A NaN (an output the kernel never
    wrote keeps the NaN it was filled with) is out of bounds."""
    err = (got - ref).abs()
    lim = r * ref.abs() + a * absb + 1e-300
    bad = ~(err <= lim)
    if mask is not None:
        bad &= mask
    if bool(bad.any()):
        worst = int(torch.where(bad, (err - lim).nan_to_num(float("inf")), -1.0).flatten().argmax())
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), got.shape))
        pytest.fail("%s: %d of %d elements out of bounds; worst at %s: got %.10g ref %.10g bound %.3g"
                    % (what, int(bad.sum()), bad.numel(), idx, float(got[idx]), float(ref[idx]), float(lim[idx])))


def ncdhw(v):
    return v.permute(0, 4, 1, 2, 3)


def ndhwc(v):
    return v.permute(0, 2, 3, 4, 1)


def chan_sums(v):
    return v.sum(dim=(1, 2, 3))


# ------------------------------------------------------------------------------------------------------------ GroupNorm
@pytest.mark.parametrize("case", B.GN_CASES, ids=lambda c: c.id)
def test_groupnorm_apply_backward_finalize(L, case):
    o = case.opt
    n, c, dims, split = case.n, case.c, case.dims, case.split
    real = o.get("real", c)
    G = o["g"] or real
    slope = o.get("slope", 0.0)
    variant = o["bwd"]
    S = B.vol(dims)
    gen = gen_of(case.id)
    r = R_STORE[split]
    xbuf_c = c + 16                                      # x is the slice [8, 8 + c) of a wider buffer, as dx and y are
    x, xv = rand_in(L, n, c, dims, split, gen, scale=2.0, shift=0.5, c_view=xbuf_c, c0=8)
    if real < c:                                         # padded channels: exact zeros in the buffer
        x.hi[..., 8 + real:8 + c] = 0
        if split:
            x.lo[..., 8 + real:8 + c] = 0
        xv = got_of(x)
    gamma = None if variant == "nogamma" else (torch.randn(real, generator=gen, device=DEV) * 0.3 + 1)
    beta = None if variant == "nogamma" else torch.randn(real, generator=gen, device=DEV) * 0.2
    g64 = gamma.double() if gamma is not None else torch.ones(real, dtype=f64, device=DEV)
    b64 = beta.double() if beta is not None else torch.zeros(real, dtype=f64, device=DEV)
    stats = torch.stack([chan_sums(xv), chan_sums(xv * xv)], dim=-1).contiguous()
    stats[:, real:] = 7.0                                # ignored
    coef = torch.full((n, c, 4), float("nan"), device=DEV)
    ybuf, y = out_view(L, n, dims, c, split)
    L.gn_apply(x, y, stats, gamma, beta, real, G, coef, slope=slope)
    torch.cuda.synchronize()
    # coefficients: fp64, rounded once
    xr = xv[..., :real]
    xg = xr.reshape(n, S, G, real // G)
    mu = xg.mean(dim=(1, 3)).repeat_interleave(real // G, dim=1)
    var = (xg * xg).mean(dim=(1, 3)).repeat_interleave(real // G, dim=1) - mu * mu
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    A, Bc = g64 * rstd, b64 - mu * g64 * rstd
    k = coef.double()
    for i, (ref, ab) in enumerate([(A, A.abs()), (Bc, b64.abs() + (mu * A).abs()), (mu, mu.abs()), (rstd, rstd)]):
        check(k[:, :real, i], ref, ab, 2 * U, 2.0 ** -40, "coef[%d]" % i)
    assert float(k[:, real:].abs().max() if real < c else 0.0) == 0.0, "coefficients of padded channels"
    # y = act(A x + B), with the fp32 coefficients the kernel stored
    A32, B32 = k[..., 0][:, None, None, None, :], k[..., 1][:, None, None, None, :]
    z = A32 * xv + B32
    yref = torch.where(z > 0, z, z * slope)
    check(got_of(y), yref, (A32 * xv).abs() + B32.abs(), r, 4 * U, "y (slope %g)" % slope)
    untouched(ybuf, c)
    # reference y through torch's own group_norm (independent of the coefficients)
    zt = ndhwc(F.group_norm(ncdhw(xr), G, g64, b64, 1e-5))
    mu_a = (mu * A)[:, None, None, None, :]
    check(z[..., :real], zt, (A32 * xv).abs()[..., :real] + B32.abs()[..., :real] + mu_a.abs(), 0.0, 8 * U, "A x + B against group_norm")
    # the first block's norm: (E, F) of dx = A dz + E x + F, dgamma and dbeta, without dx
    dz, dzv = rand_in(L, n, c, dims, split, gen)
    xq = ncdhw(xr).clone().requires_grad_(True)
    gq = g64.clone().requires_grad_(True)
    bq = b64.clone().requires_grad_(True)
    F.group_norm(xq, G, gq, bq, 1e-5).backward(ncdhw(dzv[..., :real]))
    mu32, rstd32 = k[:, :real, 2], k[:, :real, 3]
    xhat = (xr - mu32[:, None, None, None]) * rstd32[:, None, None, None]
    bst = torch.zeros(n, c, 2, dtype=f64, device=DEV)
    bst[:, :real] = torch.stack([chan_sums(dzv[..., :real]), chan_sums(dzv[..., :real] * xhat)], dim=-1)
    coef2 = torch.full((n, c, 2), float("nan"), device=DEV)
    dg2, db2 = torch.full((real,), float("nan"), device=DEV), torch.full((real,), float("nan"), device=DEV)
    L.gn_bwd_finalize(bst, coef, gamma, n, real, c, G, S, coef2, dg2, db2)
    torch.cuda.synchronize()
    c12 = (bst[:, :real] * g64[None, :, None]).reshape(n, G, real // G, 2).sum(2).repeat_interleave(real // G, dim=1) / (S * (real // G))
    E = -rstd32 * rstd32 * c12[..., 1]
    Fr = -rstd32 * c12[..., 0] + rstd32 * rstd32 * c12[..., 1] * mu32
    k2 = coef2.double()
    check(k2[:, :real, 0], E, E.abs(), 2 * U, 2.0 ** -40, "coef2 E")
    check(k2[:, :real, 1], Fr, (rstd32 * c12[..., 0]).abs() + (rstd32 * rstd32 * c12[..., 1] * mu32).abs(), 2 * U, 2.0 ** -40, "coef2 F")
    if real < c:
        assert float(k2[:, real:].abs().max()) == 0.0, "coef2 of padded channels"
    # dgamma, dbeta: the fp64 sums over the batch of the statistics the kernel was given, rounded once (autograd's dgamma takes xhat
    # from the exact mu and rstd, the statistics from the stored fp32 ones; dbeta does not depend on them)
    check(dg2.double(), bst[:, :real, 1].sum(0), bst[:, :real, 1].abs().sum(0), 2 * U, 2.0 ** -40, "dgamma (finalize)")
    check(db2.double(), bq.grad, bst[:, :real, 0].abs().sum(0), 2 * U, 2.0 ** -40, "dbeta (finalize)")
    # dx = (A dz + E x + F (+ add1) (+ add2)) * scale: against autograd of torch's group_norm; add1 is a channel slice, or a whole
    # buffer as SegResNet's ResBlocks hand over their output gradient
    ref = torch.zeros(n, *dims, c, dtype=f64, device=DEV)
    ref[..., :real] = ndhwc(xq.grad)
    absb = (A32 * dzv).abs()
    absb[..., :real] += (k2[:, None, None, None, :real, 0] * xr).abs() + k2[:, None, None, None, :real, 1].abs()
    kw = {}
    if "add1" in variant:
        a1, a1v = rand_in(L, n, c, dims, split, gen) if o.get("whole") else rand_in(L, n, c, dims, split, gen, c_view=c + 8, c0=8)
        kw["add1"] = a1
        ref, absb = ref + a1v, absb + a1v.abs()
    if "add2" in variant:
        a2, a2v = rand_in(L, n, c, dims, split, gen)
        kw["add2"] = a2
        ref, absb = ref + a2v, absb + a2v.abs()
    if "scale" in variant:
        kw["scale"] = torch.tensor([0.0, 0.8, 1.25], device=DEV)[torch.randint(0, 3, (n, c), generator=gen, device=DEV)]
        s = kw["scale"].double()[:, None, None, None, :]
        ref, absb = ref * s, absb * s
    dxbuf, dx = out_view(L, n, dims, c, split)
    dg = torch.full((real,), float("nan"), device=DEV)
    db = torch.full((real,), float("nan"), device=DEV)
    L.gn_bwd(dz, x, coef, bst, gamma, real, G, dx, dg, db, **kw)
    torch.cuda.synchronize()
    check(got_of(dx), ref, absb, r, 16 * U, "dx (%s)" % variant)
    untouched(dxbuf, c)
    assert torch.equal(dg, dg2) and torch.equal(db, db2), "dgamma / dbeta of gn_bwd and gn_bwd_finalize"


def test_groupnorm_refusals(L):
    x = L.Act.empty(1, 2, 2, 2, 1032)
    st = torch.zeros(1, 1032, 2, dtype=f64, device=DEV)
    coef = torch.zeros(1, 1032, 4, device=DEV)
    with pytest.raises(RuntimeError, match=r"status -2\).*C <= 1024 supported \(got 1032\)"):
        L.gn_apply(x, x, st, None, None, 1032, 8, coef)
    with pytest.raises(RuntimeError, match=r"status -2\).*C <= 1024 supported \(got 1032\)"):
        L.gn_bwd(x, x, coef, st, None, 1032, 8, x)
    y = L.Act.empty(1, 2, 2, 2, 24)
    for fn in (lambda: L.gn_apply(y, y, st, None, None, 24, 5, coef), lambda: L.gn_bwd(y, y, coef, st, None, 24, 5, y),
               lambda: L.gn_bwd_finalize(st, coef, None, 1, 24, 24, 5, 8, coef, None, None)):
        with pytest.raises(RuntimeError, match=r"status -1\).*C=24 G=5"):
            fn()


# -------------------------------------------------------------------------------------------------- activation backward
def _coef_of(xv, gen):
    """fp32 (A, B, mu, rstd) [n][c][4] of an instance norm of xv with random gamma / beta, and its exact fp64 value"""
    mu = xv.mean(dim=(1, 2, 3))
    rstd = 1.0 / torch.sqrt(xv.var(dim=(1, 2, 3), unbiased=False) + 1e-5)
    c = xv.shape[-1]
    gamma = (torch.randn(c, generator=gen, device=DEV) * 0.3 + 1).double()
    beta = (torch.randn(c, generator=gen, device=DEV) * 0.2).double()
    coef = torch.stack([gamma * rstd, beta - mu * gamma * rstd, mu, rstd], dim=-1).float().contiguous()
    return coef, coef.double()


@pytest.mark.parametrize("case", B.ACT_CASES, ids=lambda c: c.id)
def test_activation_backward(L, case):
    """dz = (g1 [+ g2]) * act'(A c + B) and bstats += (sum dz, sum dz * xhat), the statistics at a pitch of C + ld"""
    o = case.opt
    n, c, dims, split, slope = case.n, case.c, case.dims, case.split, o["slope"]
    ld = c + o.get("ld", 0)
    gen = gen_of(case.id)
    x, xv = rand_in(L, n, c, dims, split, gen, scale=2.0, shift=0.5)
    g1, g1v = rand_in(L, n, c, dims, split, gen)
    g2, g2v = rand_in(L, n, c, dims, split, gen) if o["g2"] else (None, 0.0)
    coef, k = _coef_of(xv, gen)
    bst = torch.full((n, ld, 2), SENTINEL, dtype=f64, device=DEV)
    bst[:, :c] = 0
    dzbuf, dz = out_view(L, n, dims, c, split)
    L.act_bwd(g1, g2, x, coef, slope, dz, bst, ld)
    torch.cuda.synchronize()
    A, Bc, mu, rstd = (k[..., i][:, None, None, None, :] for i in range(4))
    z = A * xv + Bc
    zabs = (A * xv).abs() + Bc.abs()
    clear = z.abs() > 2.0 ** -20 * zabs              # the fp32 A x + B decides the sign of these exactly as fp64 does
    g = g1v + g2v
    gabs = g1v.abs() + (g2v.abs() if o["g2"] else 0.0)
    ref = torch.where(z > 0, g, g * slope)
    check(got_of(dz), ref, gabs, R_STORE[split], 2 * U, "dz", mask=clear)
    untouched(dzbuf, c)
    # statistics: each thread sums `chain` voxels in fp32
    blocks, threads, _, _ = B.act_bwd_geometry(n, c, dims)
    vper = threads // (c // 8)
    chain = -(-B.vol(dims) // (blocks * vper)) + 2
    xhat = (xv - mu) * rstd
    amb = (~clear).double() * gabs                   # an undecided sign moves that element's dz by at most |g|
    e = 2 * U * gabs + amb
    s1 = chan_sums(ref)
    b1 = chan_sums(e) + chain * U * chan_sums(ref.abs())
    s2 = chan_sums(ref * xhat)
    b2 = chan_sums(e * xhat.abs() + ref.abs() * 4 * U * ((xv.abs() + mu.abs()) * rstd)) + chain * U * chan_sums((ref * xhat).abs())
    b = bst[:, :c]
    assert bool(((b[..., 0] - s1).abs() <= b1).all()), "sum dz: worst excess %g" % float(((b[..., 0] - s1).abs() - b1).max())
    assert bool(((b[..., 1] - s2).abs() <= b2).all()), "sum dz * xhat: worst excess %g" % float(((b[..., 1] - s2).abs() - b2).max())
    assert bool((bst[:, c:] == SENTINEL).all()), "statistics written beyond C in a pitch of %d" % ld


# ------------------------------------------------------------------------------------------------------ x2 up-sampling
def _up(v):
    return ndhwc(F.interpolate(ncdhw(v), scale_factor=2, mode="trilinear", align_corners=False))


@pytest.mark.parametrize("case", B.UP_FWD_CASES, ids=lambda c: c.id)
def test_upsample_forward_into_concat_slice(L, case):
    """y = trilinear x2 of x into channels [8, 8 + C) of a concat buffer, with the per-channel (sum, sumsq) of the fp32 values at
    a pitch of the buffer's width"""
    n, c, dims, split = case.n, case.c, case.dims, case.split
    gen = gen_of(case.id)
    x, xv = rand_in(L, n, c, dims, split, gen, shift=0.25)
    od = tuple(2 * d for d in dims)
    ybuf, y = out_view(L, n, od, c, split)
    ld = C0 + c + 8
    stats = torch.zeros(n, ld, 2, dtype=f64, device=DEV)
    stats[:, :C0] = SENTINEL
    stats[:, C0 + c:] = SENTINEL
    L.upsample2x_fwd(x, y, stats[:, C0:], ld)
    torch.cuda.synchronize()
    ref, absb = _up(xv), _up(xv.abs())
    check(got_of(y), ref, absb, R_STORE[split], 8 * U, "y")
    untouched(ybuf, c)
    blocks, threads, _, _ = B.upsample_fwd_geometry(n, c, dims)
    vper = threads // (c // 8)
    nblk = (dims[0] + 1) * (dims[1] + 1) * (dims[2] + 1)
    chain = 8 * -(-nblk // (blocks * vper)) + 6      # 8 outputs per 2 x 2 x 2 block, then at most 5 shuffle steps
    e = 8 * U * absb
    st = stats[:, C0:C0 + c]
    b1 = chan_sums(e) + chain * U * chan_sums(absb)
    b2 = chan_sums(2 * ref.abs() * e + e * e) + chain * U * chan_sums(ref * ref)
    assert bool(((st[..., 0] - chan_sums(ref)).abs() <= b1).all()), "per-channel sums"
    assert bool(((st[..., 1] - chan_sums(ref * ref)).abs() <= b2).all()), "per-channel sums of squares"
    assert bool((stats[:, :C0] == SENTINEL).all() and (stats[:, C0 + c:] == SENTINEL).all()), "statistics outside the slice"


def test_upsample_forward_refuses_more_than_2048_channels(L):
    x = L.Act.empty(1, 1, 1, 1, 2056)
    y = L.Act.empty(1, 2, 2, 2, 2056)
    with pytest.raises(RuntimeError, match=r"status -2\).*C=2056"):
        L.upsample2x_fwd(x, y)


def check_upsample_skip_add(L, n, c, dims, split, gen):
    """y = trilinear x2 of p + skip into a whole buffer, and the per-channel (sum, sumsq) of y"""
    od = tuple(2 * d for d in dims)
    p, pv = rand_in(L, n, c, dims, split, gen, shift=0.25)
    s, sv = rand_in(L, n, c, od, split, gen)
    y = L.Act.empty(n, *od, c, split=split)
    stats = torch.zeros(n, c, 2, dtype=f64, device=DEV)
    L.upsample2x_fwd(p, y, stats, c, add=s)
    torch.cuda.synchronize()
    ref = _up(pv) + sv
    absb = _up(pv.abs()) + sv.abs()
    check(got_of(y), ref, absb, R_STORE[split], 10 * U, "y")
    # statistics: the fp32 values before storage, summed in chains of 8 per 2 x 2 x 2 block
    blocks, threads, _, _ = B.upsample_fwd_geometry(n, c, dims)
    nblk = (dims[0] + 1) * (dims[1] + 1) * (dims[2] + 1)
    chain = 8 * -(-nblk // (blocks * (threads // (c // 8)))) + 6      # 8 outputs per 2 x 2 x 2 block, then the shuffles
    e = 10 * U * absb
    s1, s2 = chan_sums(ref), chan_sums(ref * ref)
    b1 = chan_sums(e) + chain * U * chan_sums(absb)
    b2 = chan_sums(2 * ref.abs() * e + e * e) + chain * U * chan_sums(ref * ref)
    assert bool(((stats[..., 0] - s1).abs() <= b1).all()), "per-channel sums"
    assert bool(((stats[..., 1] - s2).abs() <= b2).all()), "per-channel sums of squares"


@pytest.mark.parametrize("case", B.UP_ADD_CASES, ids=lambda c: c.id)
def test_upsample_skip_add_forward_and_statistics(L, case):
    """the fused x2 up-sampling + skip-add of SegResNet's decoder, with the statistics of the sum, in every regime of the plans"""
    check_upsample_skip_add(L, case.n, case.c, case.dims, case.split, gen_of(case.id))


@pytest.mark.parametrize("case", B.UP_BWD_CASES, ids=lambda c: c.id)
def test_upsample_backward_from_concat_gradient(L, case):
    """dx = the adjoint of the x2 up-sampling, reading dy as channels [0, C) of a 2C-channel concat gradient as the UNet3D plans
    do (case.view), or from a whole C-channel buffer as SegResNet's decoder does"""
    n, c, dims, split = case.n, case.c, case.dims, case.split
    gen = gen_of(case.id)
    od = tuple(2 * d for d in dims)
    dy, dyv = rand_in(L, n, c, od, split, gen, c_view=2 * c if case.view else None)
    dxbuf, dx = out_view(L, n, dims, c, split)
    L.upsample2x_bwd(dy, dx)
    torch.cuda.synchronize()
    xq = torch.zeros(n, c, *dims, dtype=f64, device=DEV, requires_grad=True)
    F.interpolate(xq, scale_factor=2, mode="trilinear", align_corners=False).backward(ncdhw(dyv))
    ref = ndhwc(xq.grad)
    xq.grad = None
    F.interpolate(xq, scale_factor=2, mode="trilinear", align_corners=False).backward(ncdhw(dyv.abs()))
    check(got_of(dx), ref, ndhwc(xq.grad), R_STORE[split], 2.0 ** -17, "dx (%s)" % case.key[0])
    untouched(dxbuf, c)


# ------------------------------------------------------------------------------------------------------- bias gradient
@pytest.mark.parametrize("case", B.BIAS_CASES, ids=lambda c: c.id)
def test_bias_grad_visible_extents_and_repeats(L, case):
    """dbias = sum of dy over its visible voxels (the high plane, row and column one short, as the plans mask the transposed
    convolution's padded boundary), in a fixed order: two runs agree bit for bit"""
    n, c, dims, split = case.n, case.c, case.dims, case.split
    gen = gen_of(case.id)
    dy, dyv = rand_in(L, n, c, dims, split, gen, c_view=C0 + c + 8, c0=C0)
    vis = tuple(d - 1 for d in dims)
    outs = []
    for _ in range(2):
        db = torch.full((c,), float("nan"), device=DEV)
        L.bias_grad(dy, db, ext=L.diag_ext(dy_vis=vis))
        torch.cuda.synchronize()
        outs.append(db)
    assert torch.equal(outs[0], outs[1]), "the bias gradient differs between two runs"
    z = dyv[:, :vis[0], :vis[1], :vis[2]]
    blocks, threads, _, _ = B.bias_grad_geometry(n, c, dims)
    vper = threads // (c // 8)
    chain = -(-n * B.vol(dims) // (blocks * vper)) + vper + -(-blocks // 128) + 8
    check(outs[0].double(), z.sum(dim=(0, 1, 2, 3)), z.abs().sum(dim=(0, 1, 2, 3)), 0.0, chain * U, "dbias")


# -------------------------------------------------------------------------------------------------------------- head
@pytest.mark.parametrize("case", B.HEAD_BWD_CASES, ids=lambda c: c.id)
def test_head_backward(L, case):
    """dx = sum_o dlogits_o w_o into a channel view, dw = sum over voxels of dlogits x (fixed order: bit for bit over two runs)"""
    n, c, dims, split, no = case.n, case.c, case.dims, case.split, case.opt["o"]
    gen = gen_of(case.id)
    x, xv = rand_in(L, n, c, dims, split, gen, c_view=c + 16, c0=8)
    w = torch.randn(no, c, generator=gen, device=DEV) * 0.3
    dl = torch.randn(n, no, *dims, generator=gen, device=DEV)
    outs = []
    for _ in range(2):
        dxbuf, dx = out_view(L, n, dims, c, split)
        dw = torch.full((no, c), float("nan"), device=DEV)
        L.head_bwd(x, w, no, dl, dx, dw)
        torch.cuda.synchronize()
        outs.append((dxbuf, dx, dw))
    assert torch.equal(outs[0][2], outs[1][2]), "head dw differs between two runs"
    dxbuf, dx, dw = outs[0]
    dlv, wv = ndhwc(dl.double()), w.double()
    check(got_of(dx), dlv @ wv, dlv.abs() @ wv.abs(), R_STORE[split], (no + 1) * U, "dx")
    untouched(dxbuf, c)
    blocks, threads, _, _ = B.head_bwd_geometry(n, c, dims)
    chain = -(-n * B.vol(dims) * (c // 8) // (blocks * threads)) + threads // (c // 8) + -(-blocks // 128) + 8
    ref = torch.einsum("ndhwo,ndhwc->oc", dlv, xv)
    check(dw.double(), ref, torch.einsum("ndhwo,ndhwc->oc", dlv.abs(), xv.abs()), 0.0, chain * U, "dw")


@pytest.mark.parametrize("case", B.HEAD_FWD_CASES, ids=lambda c: c.id)
def test_head_forward_at_plan_geometries(L, case):
    """logits = w x (+ b) of the SIMT head at the plans' grids, clamped ones with a partial last sweep included"""
    n, c, dims, split, no = case.n, case.c, case.dims, case.split, case.opt["o"]
    gen = gen_of(case.id)
    x, xv = rand_in(L, n, c, dims, split, gen)
    w = torch.randn(no, c, generator=gen, device=DEV) * 0.3
    bias = torch.randn(no, generator=gen, device=DEV)
    for b in (None, bias):
        zref = ndhwc_to_out(xv @ w.double().t() + (b.double() if b is not None else 0))
        zabs = ndhwc_to_out(xv.abs() @ w.double().abs().t() + (b.double().abs() if b is not None else 0))
        logits = torch.full((n, no, *dims), float("nan"), device=DEV)
        L.head_fwd_ex(x, w, b, no, 0, logits)
        torch.cuda.synchronize()
        check(logits.double(), zref, zabs, 0.0, (c + 2) * U, "logits (bias %s)" % (b is not None))


def head_dbias_chain(dims):
    """values a thread of k_head_dbias adds in fp32 per sample (its sweeps), plus one"""
    blocks, threads, _, _ = B.head_dbias_geometry(1, dims)
    return -(-B.vol(dims) // (blocks * threads)) + 1


@pytest.mark.parametrize("case", B.HEAD_DBIAS_CASES, ids=lambda c: c.id)
def test_head_bias_gradient_at_plan_geometries(L, case):
    """dbias = the sum of dlogits over samples and voxels, at the plans' grids: 128 blocks per output and hundreds of sweeps at
    224 x 224 x 144, a partial last sweep, one sample and several"""
    n, dims, no = case.n, case.dims, case.opt["o"]
    dl = torch.randn(n, no, *dims, generator=gen_of(case.id), device=DEV) + 0.5
    db = torch.full((no,), float("nan"), device=DEV)
    L.head_dbias(dl, db)
    torch.cuda.synchronize()
    d = dl.double()
    check(db.double(), d.sum(dim=(0, 2, 3, 4)), d.abs().sum(dim=(0, 2, 3, 4)), U, head_dbias_chain(dims) * U, "head dbias")


@pytest.mark.parametrize("c", [8, 24, 32, 48, 64])
@pytest.mark.parametrize("n_out", range(1, 9))
def test_head_forward_bias_and_epilogues(L, n_out, c):
    """logits = act(w x + b) for every SIMT instance (1..8 outputs), act 0 (none), 1 (sigmoid), 2 (softmax over outputs), with and
    without a bias, from an 8-channel-offset view; and the bias gradient against an fp64 sum"""
    gen = gen_of("head%d-%d" % (n_out, c))
    n, dims, split = 2, (6, 6, 10), c % 16 == 8
    x, xv = rand_in(L, n, c, dims, split, gen, c_view=c + 16, c0=8)
    w = torch.randn(n_out, c, generator=gen, device=DEV) * 0.3
    bias = torch.randn(n_out, generator=gen, device=DEV)
    for b in (None, bias):
        zref = ndhwc_to_out(xv @ w.double().t() + (b.double() if b is not None else 0))
        zabs = ndhwc_to_out(xv.abs() @ w.double().abs().t() + (b.double().abs() if b is not None else 0))
        ez = (c + 2) * U * zabs
        for act in (0, 1, 2):
            logits = torch.full((n, n_out, *dims), float("nan"), device=DEV)
            L.head_fwd_ex(x, w, b, n_out, act, logits)
            torch.cuda.synchronize()
            got = logits.double()
            what = "n_out %d act %d bias %s" % (n_out, act, b is not None)
            if act == 0:
                check(got, zref, zabs, 0.0, (c + 2) * U, what)
            elif act == 1:
                p = torch.sigmoid(zref)
                check(got, p, 0.25 * ez + 2.0 ** -19 * p, 0.0, 1.0, what)
            else:
                p = torch.softmax(zref, dim=1)
                check(got, p, p * (2 * ez.amax(dim=1, keepdim=True) + 2.0 ** -18), 0.0, 1.0, what)
    dl = torch.randn(n, n_out, *dims, generator=gen, device=DEV)
    db = torch.full((n_out,), float("nan"), device=DEV)
    L.head_dbias(dl, db)
    torch.cuda.synchronize()
    d = dl.double()
    check(db.double(), d.sum(dim=(0, 2, 3, 4)), d.abs().sum(dim=(0, 2, 3, 4)), U, head_dbias_chain(dims) * U, "head dbias")


def ndhwc_to_out(v):
    """[n, d, h, w, o] -> [n, o, d, h, w]"""
    return v.permute(0, 4, 1, 2, 3)


# ------------------------------------------------------------------------------------------------------- zero insertion
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("off,extra", [((0, 0, 0), (0, 0, 0)), ((1, 0, 1), (0, 0, 0)), ((0, 0, 0), (2, 1, 3)), ((1, 0, 1), (1, 2, 0))])
def test_zero_insert(L, off, extra, split):
    """z[2d + od][2h + oh][2w + ow] = x[d][h][w], zeros elsewhere, over a z at least 2x - 1 + offset long, into a channel view"""
    gen = gen_of("zi%s%s%d" % (off, extra, split))
    n, c, dims = 2, 24, (3, 4, 5)
    x, xv = rand_in(L, n, c, dims, split, gen, c_view=c + 8, c0=8)
    zd = tuple(2 * d - 1 + o + e for d, o, e in zip(dims, off, extra))
    zbuf, z = out_view(L, n, zd, c, split)
    L.zero_insert(x, z, *off)
    torch.cuda.synchronize()
    ref = torch.zeros(n, *zd, c, dtype=f64, device=DEV)
    ref[:, off[0]::2, off[1]::2, off[2]::2][:, :dims[0], :dims[1], :dims[2]] = xv
    assert torch.equal(got_of(z), ref)
    untouched(zbuf, c)


# ------------------------------------------------------------------------------------------- network input: pack, gradient
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("c", list(range(1, 17)))
def test_input_pack(L, c, split):
    """NCDHW fp32 -> NDHWC bf16 (round to nearest even, lo = bf16(x - hi)) in an 8- or 16-channel view, padded channels exactly
    zero, and the fp64 (sum, sumsq) of each channel; S = 7 * 9 * 11 is not a multiple of the 256-voxel block"""
    gen = gen_of("pack%d%d" % (c, split))
    n, dims = 2, (7, 9, 11)
    cp = 8 if c <= 8 else 16
    x = torch.randn(n, c, *dims, generator=gen, device=DEV) * 3 + 0.5
    buf, out = out_view(L, n, dims, cp, split)
    ld = c + 8
    stats = torch.full((n, ld, 2), SENTINEL, dtype=f64, device=DEV)
    stats[:, :c] = 0
    L.input_pack(x, out, stats, ld)
    torch.cuda.synchronize()
    v = ndhwc(x)
    hi = v.bfloat16()
    assert torch.equal(out.hi[..., C0:C0 + c], hi), "hi is torch's round to nearest even"
    assert bool((out.hi[..., C0 + c:C0 + cp] == 0).all()), "padded channels"
    if split:
        assert torch.equal(out.lo[..., C0:C0 + c], (v - hi.float()).bfloat16()), "lo = bf16(x - hi)"
        assert bool((out.lo[..., C0 + c:C0 + cp] == 0).all())
    untouched(buf, cp)
    S = B.vol(dims)
    blocks = min(-(-S // 256), 1184)
    chain = -(-S // (blocks * 256)) + 5
    xd = v.double()
    for j, (ref, ab) in enumerate([(chan_sums(xd), chan_sums(xd.abs())), (chan_sums(xd * xd), chan_sums(xd * xd))]):
        assert bool(((stats[:, :c, j] - ref).abs() <= chain * U * ab).all()), "input statistics %d" % j
    assert bool((stats[:, c:] == SENTINEL).all())


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("c", [1, 4, 8, 9, 16])
@pytest.mark.parametrize("norm", [False, True])
def test_input_grad(L, c, norm, split):
    """dx NCDHW fp32 = (A dz + E x + F) + r from 8- or 16-channel views; without the norm step dx = r exactly"""
    gen = gen_of("igrad%d%d%d" % (c, norm, split))
    n, dims = 2, (5, 9, 13)                       # S = 585: the last 256-voxel tile is partial
    cp = 8 if c <= 8 else 16
    r, rv = rand_in(L, n, cp, dims, split, gen, c_view=cp + 16, c0=8)
    dx = torch.full((n, c, *dims), float("nan"), device=DEV)
    if not norm:
        L.input_grad(None, None, None, None, 0, r, c, dx)
        torch.cuda.synchronize()
        assert torch.equal(dx.double(), ncdhw(rv[..., :c])), "dx = r"
        return
    dz, dzv = rand_in(L, n, cp, dims, split, gen, c_view=cp + 8, c0=8)
    x, xv = rand_in(L, n, cp, dims, split, gen, shift=0.5)
    ld = cp + 8
    coef = torch.randn(n, ld, 4, generator=gen, device=DEV)
    coef2 = torch.randn(n, ld, 2, generator=gen, device=DEV)
    L.input_grad(dz, x, coef, coef2, ld, r, c, dx)
    torch.cuda.synchronize()
    a = coef[:, None, None, None, :c, 0].double()
    e, f = coef2[:, None, None, None, :c, 0].double(), coef2[:, None, None, None, :c, 1].double()
    ref = a * dzv[..., :c] + e * xv[..., :c] + f + rv[..., :c]
    absb = (a * dzv[..., :c]).abs() + (e * xv[..., :c]).abs() + f.abs() + rv[..., :c].abs()
    check(ndhwc(dx.double()), ref, absb, 0.0, 4 * U, "dx")


# -------------------------------------------------------------------------------------------------------- converters
@pytest.mark.parametrize("split", [False, True])
def test_layout_converters(L, split):
    """ncdhw_to_ndhwc rounds exactly as torch does (hi, and lo = bf16(x - hi)) and zeroes the padded channels; ndhwc_to_ncdhw is
    exact, reads c_real < c channels, and reads channel slices"""
    lib = L.load_library()
    gen = gen_of("conv%d" % split)
    n, c, dims = 2, 13, (3, 5, 6)
    x = torch.randn(n, c, *dims, generator=gen, device=DEV) * 5
    a = L.Act.empty(n, *dims, 16, split=split)
    a.hi.fill_(SENTINEL)
    if split:
        a.lo.fill_(SENTINEL)
    L.check(lib.b200unet_ncdhw_to_ndhwc(x.data_ptr(), c, L.C.byref(a.ct()), L.stream_ptr()), "ncdhw_to_ndhwc")
    torch.cuda.synchronize()
    v = ndhwc(x)
    hi = v.bfloat16()
    assert torch.equal(a.hi[..., :c], hi) and bool((a.hi[..., c:] == 0).all())
    if split:
        assert torch.equal(a.lo[..., :c], (v - hi.float()).bfloat16()) and bool((a.lo[..., c:] == 0).all())
    # back: a slice of 8 channels at offset 8 of a 24-channel buffer, 5 of them read
    src, sv = rand_in(L, n, 8, dims, split, gen, c_view=24, c0=8)
    y = torch.full((n, 5, *dims), float("nan"), device=DEV)
    L.check(lib.b200unet_ndhwc_to_ncdhw(L.C.byref(src.ct()), 5, y.data_ptr(), L.stream_ptr()), "ndhwc_to_ncdhw")
    torch.cuda.synchronize()
    assert torch.equal(y.double(), ncdhw(sv[..., :5]))
