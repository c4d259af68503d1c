"""The tensor-core head for 9..128 outputs (csrc/head.cu) against fp64, element by element, at the launch geometries of
tests/head_cases.py: logits, dx, dw and the fused bias gradient.

x is bf16 hi (+ lo in split precision), so its fp64 value is exact; w, bias and dlogits are fp32; the references run on the
device in fp64.  Every element must satisfy |got - ref| <= bound, with the bound fixed by a model of the kernels' arithmetic,
never by what a GPU shows (A = the sum of the products' magnitudes, u = 2^-24):
  - products: split precision drops lo*lo and leaves a residual of each two-term split, each at most 2^-16 |a||b| per split
    operand (x is exact: forward and dw split one operand, dx splits w and dlogits); bf16 mode rounds w (and dlogits in the
    backward), 2^-8 |a||b| per rounded operand;
  - accumulation: chain * u * A, the chain counting 16 products per k16 step per MMA pass (3 passes in split precision):
    forward 16 ceil(C / 16), dx 16 NT; dw 128 voxels x its CTA's tiles, plus k_sum_slots' ceil(slots / 128) + 7; dbias its
    CTA's tiles + 2 (a thread's voxel quad) + 2 shuffles + 8 warps + the slot sum;
  - dx is stored as bf16 hi + lo (2^-17 relative) or bf16 (2^-8); the bias add and the final rounding one u each;
  - sigmoid and softmax through __expf: relative (6 + 1.2 |r|) u and (n_out + 6 + 4.5 max_o |r|) u (the model of
    tests/test_gpu_loss_prepost_kernels.py), plus the logit error through the Jacobian.
The positive rows make A = |value| for dw and dbias, so a lost tile shows above the chain bound where a CTA walks few tiles:
on the 2 x 32 x 33 x 32 rows (4 per backward slot) it is a quarter of the sum.  At the C2 size (249 tiles per slot) the dw
chain bound is 0.57 % of the sum, above the 0.40 % one lost tile per CTA would cost, so there the rows hold dw to the chain
bound only and the cross-tile accumulation is checked by the smaller multi-tile rows.  Buffers around every output
hold NaN sentinels that must survive, the backward scratch is NaN-filled and must hold exactly the restated slots, reruns must
repeat bit for bit, and dlogits at a one-float offset must give the aligned run's bits.
"""
import time
import zlib

import pytest
import torch

import head_cases as H

pytestmark = pytest.mark.gpu

DEV = "cuda"
f64 = torch.float64
U = H.U
ACT_ID = {"none": 0, "sigmoid": 1, "softmax": 2}
PAD = 64                      # sentinel floats before and after the logits
REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    t0 = time.time()
    yield
    print("\nobserved error as a fraction of its bound (worst element):")
    for k, v in sorted(REPORT.items()):
        print("  %-60s %s" % (k, "  ".join("%s %.3f" % kv for kv in sorted(v.items()))))
    print("test_gpu_head_kernels: %.1f s" % (time.time() - t0))


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


# ------------------------------------------------------------------------------------------------------------- inputs
def _x(pkg, case, gen):
    """x as a channel view [c0, c0 + c) of an NDHWC tensor with ld channels (NaN outside the view); its exact fp64 value
    [n][S][c]"""
    n, c, split = case.n, case.c, case.precision == "split"
    ld, c0 = (case.ld, 8) if case.ld else (c, 0)
    v = torch.randn((n,) + case.dims + (c,), generator=gen, device=DEV)
    if case.positive:
        v = v.abs() + 0.05
    hi = v.to(torch.bfloat16)
    lo = (v - hi.float()).to(torch.bfloat16) if split else None
    val = (hi.double() + (lo.double() if split else 0)).reshape(n, -1, c)
    del v

    def wide(t):
        if t is None:
            return None
        full = torch.full((n,) + case.dims + (ld,), float("nan"), dtype=torch.bfloat16, device=DEV)
        full[..., c0:c0 + c] = t
        return full
    return pkg.lib.Act(wide(hi), wide(lo), c0, c), val


def _dx_buffers(pkg, case):
    """dx as the same channel view, inside NaN-filled storage one sample longer"""
    ld, c0 = (case.ld, 8) if case.ld else (case.c, 0)
    shape = (case.n + 1,) + case.dims + (ld,)
    hi = torch.full(shape, float("nan"), dtype=torch.bfloat16, device=DEV)
    lo = torch.full(shape, float("nan"), dtype=torch.bfloat16, device=DEV) if case.precision == "split" else None
    return pkg.lib.Act(hi[:case.n], lo[:case.n] if lo is not None else None, c0, case.c), (hi, lo, c0)


def _untouched(full, n, c0, c, what):
    rest = full.clone()
    rest[:n, ..., c0:c0 + c] = float("nan")
    assert bool(torch.isnan(rest).all()), "%s: written outside its view" % what


def _dlogits(case, gen):
    shape = (case.n, case.n_out) + case.dims
    return torch.rand(shape, generator=gen, device=DEV) + 0.05 if case.positive else torch.randn(shape, generator=gen, device=DEV)


def _at_offset(g, off):
    buf = torch.zeros(g.numel() + 8, device=DEV)
    buf[off:off + g.numel()] = g.flatten()
    return buf[off:off + g.numel()].view(g.shape)


# ---------------------------------------------------------------------------------------------------------- forward
def _forward(pkg, case, x, w, bias):
    numel = case.n * case.n_out * case.geometry["S"]
    buf = torch.full((PAD + numel + PAD,), float("nan"), device=DEV)
    logits = buf[PAD:PAD + numel].view((case.n, case.n_out) + case.dims)
    pkg.lib.head_fwd_ex(x, w, bias, case.n_out, ACT_ID[case.act], logits)
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[:PAD]).all() and torch.isnan(buf[PAD + numel:]).all()), "logits: written outside the tensor"
    return logits


def _check_forward(case, logits, xval, w, bias):
    g = case.geometry
    split = case.precision == "split"
    npass = 3 if split else 1
    w64, wa = w.double(), w.double().abs()
    worst = 0.0
    for n in range(case.n):
        r = xval[n] @ w64.T                                              # [S][n_out]
        A = xval[n].abs() @ wa.T
        if bias is not None:
            r += bias.double()
            A += bias.double().abs()
        prod = (2 * 2.0 ** -16 if split else 2.0 ** -8) * A
        dr = prod + (16 * g["ksteps"] * npass + 2) * U * A + U * r.abs()
        if case.act == "none":
            ref, lim = r, dr
        elif case.act == "sigmoid":
            ref = torch.sigmoid(r)
            lim = ref * (1 - ref) * dr + (6 + 1.2 * r.abs()) * U * ref
        else:
            ref = torch.softmax(r, 1)
            X = r.abs().amax(1, keepdim=True)
            lim = ref * (dr + (ref * dr).sum(1, keepdim=True)) + (case.n_out + 6 + 4.5 * X) * U * ref
        del A, r
        worst = max(worst, within(logits[n].reshape(case.n_out, -1).T, ref, lim * 1.01 + 1e-30, "%s logits sample %d" % (case.id, n)))
    note(case, "logits", worst)


@pytest.mark.parametrize("case", H.CASES, ids=lambda c: c.id)
def test_head_forward_and_backward_match_fp64(pkg, case):
    L = pkg.lib
    gen = gen_of(case.id)
    geo = case.geometry
    x, xval = _x(pkg, case, gen)
    w = torch.randn(case.n_out, case.c, generator=gen, device=DEV) / case.c ** 0.5
    bias = torch.randn(case.n_out, generator=gen, device=DEV) * 0.5 if case.bias else None

    # forward: against fp64, then a rerun repeats it bit for bit
    logits = _forward(pkg, case, x, w, bias)
    _check_forward(case, logits, xval, w, bias)
    assert torch.equal(_forward(pkg, case, x, w, bias), logits), "%s: forward rerun differs" % case.id
    del logits

    # backward
    g = _dlogits(case, gen)
    g_in = _at_offset(g, case.offset) if case.offset else g
    assert (g_in.data_ptr() % 16 != 0) == (geo["path"] == "unaligned")
    scratch_floats = L.head_bwd_scratch_bytes(case.n_out, case.c) // 4

    def backward(gl):
        dx, (hi, lo, c0) = _dx_buffers(pkg, case)
        dw = torch.full((case.n_out, case.c), float("nan"), device=DEV)
        db = torch.full((case.n_out,), float("nan"), device=DEV) if case.bias else None
        scratch = torch.full((scratch_floats,), float("nan"), device=DEV)
        L.head_bwd_ex(x, w, case.n_out, gl, dx, dw, db, scratch)
        torch.cuda.synchronize()
        _untouched(hi, case.n, c0, case.c, case.id + " dx.hi")
        if lo is not None:
            _untouched(lo, case.n, c0, case.c, case.id + " dx.lo")
        # slot partials: exactly the restated slot count is written, the rest of the scratch keeps its NaN
        nc, slots = case.n_out * case.c, geo["slots"]
        used = slots * nc + (slots * case.n_out if case.bias else 0)
        assert bool(torch.isfinite(scratch[:used]).all()), "%s: a slot of the %d restated ones was not written" % (case.id, slots)
        assert bool(torch.isnan(scratch[used:]).all()), "%s: more than the %d restated slots were written" % (case.id, slots)
        return dx, dw, db

    dx, dw, db = backward(g_in)
    _check_backward(case, g, xval, w, dx, dw, db)
    runs = [backward(g_in)]
    if case.offset:
        runs.append(backward(g))                                     # the vector path must give the same bits
    def view(a, t):
        return t[..., a.c0:a.c0 + a.c]
    for dx2, dw2, db2 in runs:
        assert torch.equal(view(dx2, dx2.hi), view(dx, dx.hi)), "%s: dx differs" % case.id
        assert dx.lo is None or torch.equal(view(dx2, dx2.lo), view(dx, dx.lo)), "%s: dx differs" % case.id
        assert torch.equal(dw2, dw), "%s: dw differs" % case.id
        assert db is None or torch.equal(db2, db), "%s: dbias differs" % case.id


def _check_backward(case, g, xval, w, dx, dw, db):
    geo = case.geometry
    split = case.precision == "split"
    npass = 3 if split else 1
    w64, wa = w.double(), w.double().abs()
    slot_chain = H.cdiv(geo["slots"], 128) + 7
    e_dx = 3 * 2.0 ** -16 if split else 2 * 2.0 ** -8 + 2.0 ** -16
    e_dw = 2 * 2.0 ** -16 if split else 2.0 ** -8
    store = 2.0 ** -17 if split else 2.0 ** -8
    dw_ref = torch.zeros(case.n_out, case.c, dtype=f64, device=DEV)
    dw_abs = torch.zeros_like(dw_ref)
    db_ref = torch.zeros(case.n_out, dtype=f64, device=DEV)
    db_abs = torch.zeros_like(db_ref)
    worst = 0.0
    for n in range(case.n):
        gn = g[n].reshape(case.n_out, -1).double()                    # [n_out][S]
        ga = gn.abs()
        ref = gn.T @ w64                                             # [S][c]
        A = ga.T @ wa
        e = e_dx * A + 16 * geo["NT"] * npass * U * A
        lim = e + store * (ref.abs() + e)
        got = dx.hi[n][..., dx.c0:dx.c0 + case.c].double() + (dx.lo[n][..., dx.c0:dx.c0 + case.c].double() if split else 0)
        worst = max(worst, within(got.reshape(-1, case.c), ref, lim * 1.01 + 1e-30, "%s dx sample %d" % (case.id, n)))
        del ref, A, e, lim, got
        dw_ref += gn @ xval[n]
        dw_abs += ga @ xval[n].abs()
        db_ref += gn.sum(1)
        db_abs += ga.sum(1)
    note(case, "dx", worst)
    lim = (e_dw + (npass * 128 * geo["bwd_per_cta"] + slot_chain) * U) * dw_abs
    note(case, "dw", within(dw, dw_ref, lim * 1.01 + 1e-30, case.id + " dw"))
    if db is not None:
        lim = (geo["bwd_per_cta"] + 2 + 2 + 8 + slot_chain) * U * db_abs
        note(case, "dbias", within(db, db_ref, lim * 1.01 + 1e-30, case.id + " dbias"))


# ------------------------------------------------------------------------------------------------------------- plans
def _plan_grads(pkg, model, x, g, monkeypatch):
    """parameter gradients of out.backward(g), and the dlogits pointer the plan's backward handed to the library"""
    lib = pkg.lib.load_library()
    real = lib.b200unet_plan_backward
    seen = []

    def spy(handle, dlogits, *rest):
        seen.append(dlogits)
        return real(handle, dlogits, *rest)
    monkeypatch.setattr(lib, "b200unet_plan_backward", spy)
    model.zero_grad(set_to_none=True)
    model(x).backward(g)
    torch.cuda.synchronize()
    monkeypatch.setattr(lib, "b200unet_plan_backward", real)
    assert len(seen) == 1
    return {k: p.grad.clone() for k, p in model.named_parameters()}, seen[0]


@pytest.mark.parametrize("arch", ["unet3d-16", "dynunet-14-bias"])
def test_plan_backward_takes_dlogits_at_any_storage_offset(pkg, arch, monkeypatch):
    """a contiguous gradient one float into its storage (out.backward(buf[1:].view_as(out)), or a loss over a concatenation)
    reaches the plan's backward as it is (the pointer handed to the library is checked): every parameter gradient must equal
    the aligned run's bit for bit"""
    gen = torch.Generator().manual_seed(11)
    if arch == "unet3d-16":
        model = pkg.UNet3D(precision="split", deterministic=True, dropout=0.0, n_features=4, n_outputs=16, base_width=8)
    else:
        model = pkg.DynUNet(precision="split", deterministic=True, spatial_dims=3, in_channels=4, out_channels=14,
                            kernel_size=[[3, 3, 3]] * 3, strides=[[1, 1, 1]] + [[2, 2, 2]] * 2, upsample_kernel_size=[[2, 2, 2]] * 2,
                            filters=[16, 24, 32])
        with torch.no_grad():
            model.output_block.conv.conv.bias.copy_(torch.linspace(-0.5, 0.5, 14))
    model = model.to(DEV)
    model.train()
    x = torch.randn(2, 4, 16, 16, 16, generator=gen).to(DEV)
    g = torch.randn((2, 16 if arch == "unet3d-16" else 14, 16, 16, 16), generator=gen).to(DEV)
    ref, p_ref = _plan_grads(pkg, model, x, g, monkeypatch)
    assert p_ref % 16 == 0
    buf = torch.zeros(g.numel() + 1, device=DEV)
    buf[1:] = g.flatten()
    g_off = buf[1:].view_as(g)
    assert g_off.is_contiguous() and g_off.data_ptr() % 16 != 0
    got, p_off = _plan_grads(pkg, model, x, g_off, monkeypatch)
    assert p_off == g_off.data_ptr(), "the plan's backward did not receive the misaligned gradient itself"
    assert ref.keys() == got.keys()
    for k in ref:
        assert torch.isfinite(ref[k]).all(), k
        assert torch.equal(got[k], ref[k]), k
