"""The augmentation and foreground-crop kernels (csrc/augment.cu, csrc/foreground.cu) at the cases of tests/augment_cases.py,
through the C ABI, into NaN-sentinel buffers wider than their outputs:
  - the trilinear image resample element by element against the fp64 oracle, under a per-voxel bound from an error model
    (the composed affine rounded to fp32 and the three-fma coordinate chain, times the largest corner difference on each
    axis, plus the weights and the 8-term fma chain); labels exactly outside the band where that coordinate error can reach
    a rounding tie;
  - the per-block partials and the statistics within the fp64 addition chains the block counts give;
  - the intensity pass within the fp32 (x - m) * inv and fmaf roundings;
  - thresholds bit for bit with np.percentile, boxes and empty flags exactly, the composed source affine to one fp32 rounding;
  - every result bit-identical run to run.
Each case prints its worst error as a fraction of its bound."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import augment_cases as A  # noqa: E402
import augment_oracle  # noqa: E402
import geometry_oracle  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
PAD = 64                     # sentinel elements on each side of every output
U = A.U32
PADDING = {"border": 0, "zeros": 1}


@pytest.fixture(scope="module")
def lib(pkg):
    return pkg.lib.load_library()


def _padded(n, dtype, fill, offset=0):
    """(buffer, view of n elements starting PAD + offset elements in) filled with the sentinel"""
    buf = torch.full((n + 2 * PAD + offset,), fill, dtype=dtype, device=DEV)
    return buf, buf[PAD + offset:PAD + offset + n]


def _sentinels_intact(buf, view, fill):
    lo = (view.data_ptr() - buf.data_ptr()) // buf.element_size()
    rest = torch.cat([buf[:lo], buf[lo + view.numel():]])
    return bool(rest.isnan().all()) if isinstance(fill, float) and np.isnan(fill) else bool((rest == fill).all())


def _bits(t):
    return t.contiguous().view(torch.uint8).cpu()


# ------------------------------------------------------------------------------------------------------------ resample
def _rotation_affine(out, angles, flips):
    """flips then the rotation about the output grid's centre, as augment.Compose composes them: 4x4 fp64"""
    m = np.eye(4)
    for a in flips:
        f = np.eye(4)
        f[a, a], f[a, 3] = -1.0, out[a] - 1.0
        m = m @ f
    x, y, z = angles
    rx = np.array([[1, 0, 0], [0, np.cos(x), -np.sin(x)], [0, np.sin(x), np.cos(x)]])
    ry = np.array([[np.cos(y), 0, np.sin(y)], [0, 1, 0], [-np.sin(y), 0, np.cos(y)]])
    rz = np.array([[np.cos(z), -np.sin(z), 0], [np.sin(z), np.cos(z), 0], [0, 0, 1]])
    r = np.eye(4)
    r[:3, :3] = rx @ ry @ rz
    c = (np.asarray(out, dtype=np.float64) - 1) / 2
    r[:3, 3] = c - r[:3, :3] @ c
    return m @ r


def _sample_affine(out, size, a4):
    """crop box [1, size - 1) (the whole axis below 3 voxels) resized onto out, then a4: b + s (A p) + (s - 1) / 2, fp64 3x4"""
    b0 = np.array([1.0 if s >= 3 else 0.0 for s in size])
    b1 = np.array([s - 1.0 if s >= 3 else float(s) for s in size])
    s = (b1 - b0) / np.asarray(out, dtype=np.float64)
    m = a4[:3].copy() * s[:, None]
    m[:, 3] += b0 + (s - 1) / 2
    return m


def _resample_data(case):
    """per-sample fp32 images [C][d][h][w] (channel c ~ (c + 1) N(0, 1) + c, a share of exact zeros with ``nonzero``) and
    uint8 labels, and the fp64 3x4 map of each sample"""
    g = torch.Generator().manual_seed(sum(map(ord, case.id)))
    sizes = list(case.samples) if case.source == "samples" else [case.out] * case.n
    imgs, labs, maps = [], [], []
    for i, sz in enumerate(sizes):
        x = torch.randn((case.c,) + tuple(sz), generator=g) * torch.arange(1, case.c + 1).view(-1, 1, 1, 1) \
            + torch.arange(case.c).view(-1, 1, 1, 1)
        if case.nonzero:
            x[torch.rand(x.shape, generator=g) < 0.3] = 0.0
        imgs.append(x)
        labs.append((torch.rand((case.l,) + tuple(sz), generator=g) * 5).to(torch.uint8))
        a4 = _rotation_affine(case.out, [v * (1 - 0.3 * i) for v in case.angles], case.flips)
        maps.append(_sample_affine(case.out, sz, a4) if case.source == "samples" else a4[:3])
    return sizes, imgs, labs, maps


def _run_resample(lib, pkg, case, sizes, imgs, labs, maps):
    """one resample + intensity pass; returns host copies of (image after the resample, labels, partials, stats, image after
    the intensity pass, coef, sentinels intact)"""
    n, c, l, out = case.n, case.c, case.l, case.out
    S = A.vol(out)
    nb = A.aug_blocks(S)
    ok = True
    affine = torch.tensor(np.stack(maps), dtype=torch.float32).reshape(-1).to(DEV)
    obuf, o = _padded(n * c * S, torch.float32, float("nan"))
    lbuf, lo = _padded(max(n * l * S, 1), torch.uint8, 0xAB)
    nbytes = int(lib.b200unet_augment_scratch_bytes(n, c, S))
    assert nbytes == 8 * 3 * n * c * (1 + nb)
    sbuf, scratch = _padded(nbytes // 8, torch.float64, float("nan"))
    if case.source == "batch":
        x = torch.stack(imgs).to(DEV)
        lab = torch.stack(labs).to(DEV) if l else None
        st = lib.b200unet_augment_resample(x.data_ptr(), lab.data_ptr() if l else None, n, c, l, *out, affine.data_ptr(),
                                           PADDING[case.padding], int(case.nonzero), o.data_ptr(), lo.data_ptr() if l else None,
                                           scratch.data_ptr(), pkg.lib.stream_ptr())
        keep = (x, lab)
    else:
        xs = [t.to(DEV) for t in imgs]
        ls = [t.to(DEV) for t in labs]
        rows = torch.tensor([[xs[i].data_ptr(), ls[i].data_ptr() if l else 0] + list(sizes[i]) for i in range(n)],
                            dtype=torch.int64, device=DEV)
        st = lib.b200unet_augment_resample_samples(rows.data_ptr(), n, c, l, *out, affine.data_ptr(), PADDING[case.padding],
                                                   int(case.nonzero), o.data_ptr(), lo.data_ptr() if l else None,
                                                   scratch.data_ptr(), pkg.lib.stream_ptr())
        keep = (xs, ls, rows)
    pkg.lib.check(st, "augment_resample")
    torch.cuda.synchronize()
    ok &= _sentinels_intact(obuf, o, float("nan")) and (not l or _sentinels_intact(lbuf, lo, 0xAB))
    y = o.view(n, c, *out).cpu().clone()
    labels = lo[: n * l * S].view(n, l, *out).cpu().clone() if l else None
    part = scratch[3 * n * c:].view(n, nb, c, 3).cpu().clone()
    coef = torch.tensor(np.stack([np.random.default_rng(S + c).uniform(0.9, 1.1, n * c),
                                  np.random.default_rng(S - c).uniform(-0.1, 0.1, n * c)], -1), dtype=torch.float32).to(DEV)
    pkg.lib.check(lib.b200unet_augment_intensity(o.data_ptr(), n, c, S, 1, int(case.nonzero), int(case.channel_wise),
                                                 coef.data_ptr(), scratch.data_ptr(), pkg.lib.stream_ptr()), "augment_intensity")
    torch.cuda.synchronize()
    ok &= _sentinels_intact(obuf, o, float("nan")) and _sentinels_intact(sbuf, scratch, float("nan"))
    stats = scratch[: 3 * n * c].view(n, c, 3).cpu().clone()
    z = o.view(n, c, *out).cpu().clone()
    del keep
    return y, labels, part, stats, z, coef.cpu().view(n, c, 2), ok


def _dilate(a):
    """max over the window [i - 1, i + 2] on every axis (clamped): the corners of the cells a point within a voxel of cell i
    can use"""
    for ax in range(3):
        n = a.shape[ax]
        idx = np.arange(n)
        a = np.maximum.reduce([np.take(a, np.clip(idx + k, 0, n - 1), axis=ax) for k in (-1, 0, 1, 2)])
    return a


def resample_bound(vol, src, m, padding):
    """per-voxel bound on |kernel - fp64 trilinear| for one channel vol [d][h][w] (fp64) read at the fp64 source coordinates
    src [D][H][W][3] of the map m (3x4 fp64):
      coordinate error per axis  delta_a = 4 u (sum_j |m_aj| |p_j| + |m_a3|) + u: each of the four entries rounded to fp32 and
                                 each of the three fmas rounding once (both relative to that sum), and the fraction x - floor(x)
                                 rounding once below 0 (zeros padding);
      value                      sum_a delta_a G_a + 14 u M: G_a the largest difference between neighbours along axis a among
                                 the corners the point and its perturbation can use (edge-extended or zero-padded as the
                                 padding mode), M the largest corner magnitude; 14 u covers the weights (1 - f rounded, two
                                 products: 5 u) and the 8-term fma chain (8 u), plus 1 u of slack."""
    border = padding == "border"
    pv = np.pad(vol, 2, mode="edge" if border else "constant")
    D, H, W = src.shape[:3]
    p = np.stack(np.meshgrid(np.arange(D), np.arange(H), np.arange(W), indexing="ij"), -1).astype(np.float64)
    reach = np.abs(p) @ np.abs(m[:, :3]).T + np.abs(m[:, 3])
    delta = 4 * U * reach * (1 + 1e-6) + U
    x = src
    if border:
        x = np.minimum(np.maximum(x, 0), np.asarray(vol.shape, dtype=np.float64) - 1)
    idx = [np.clip(np.floor(x[..., a]).astype(np.int64) + 2, 0, pv.shape[a] - 1) for a in range(3)]
    total = 14 * U * _dilate(np.abs(pv))[idx[0], idx[1], idx[2]]
    for a in range(3):
        g = np.abs(np.diff(pv, axis=a))
        g = np.concatenate([g, np.zeros_like(np.take(g, [0], axis=a))], axis=a)
        total += delta[..., a] * _dilate(g)[idx[0], idx[1], idx[2]]
    return total + 1e-12 * (1.0 + np.abs(vol).max()), delta


def _label_ties(src, delta, size, padding):
    x = src
    if padding == "border":
        x = np.minimum(np.maximum(x, 0), np.asarray(size, dtype=np.float64) - 1)
    return (np.abs(x - np.floor(x) - 0.5) < delta + 1e-9).any(-1)


def _check_partials(y, part, case):
    """per-block partials = fp64 sums of the kernel's own output over the restated block ranges, within the block's chain"""
    n, c = case.n, case.c
    S = A.vol(case.out)
    g = A.resample_geometry(S)
    starts = np.array([r[0] for r in A.aug_block_ranges(S)])
    yv = y.view(n, c, S).double().numpy()
    worst = 0.0
    for i in range(n):
        for ch in range(c):
            v = yv[i, ch].astype(np.longdouble)
            sel = (v != 0) if case.nonzero else np.ones_like(v, dtype=bool)
            for j, terms in enumerate((v, v * v)):
                ref = np.add.reduceat(terms, starts)
                mag = np.add.reduceat(np.abs(terms), starts)
                bound = (g["block_chain"] + 1) * A.U64 * mag.astype(np.float64) + 1e-300
                err = np.abs(part[i, :, ch, j].numpy().astype(np.longdouble) - ref).astype(np.float64)
                assert (err <= bound).all(), (case.id, i, ch, j, float((err / bound).max()))
                worst = max(worst, float((err / bound).max()))
            cnt = np.add.reduceat(sel.astype(np.int64), starts)
            assert np.array_equal(part[i, :, ch, 2].numpy(), cnt.astype(np.float64)), (case.id, i, ch)
    return worst


def _check_stats(part, stats, chain):
    """stats [n][c][3] = sum over the blocks of part [n][nb][c][3], within the chain of k_aug_stats"""
    p = part.numpy().astype(np.longdouble)
    ref = p.sum(1)
    bound = (chain + 1) * A.U64 * np.abs(p).sum(1).astype(np.float64) + 1e-300
    err = np.abs(stats.numpy().astype(np.longdouble) - ref).astype(np.float64)
    assert (err[..., :2] <= bound[..., :2]).all(), float((err / bound).max())
    assert np.array_equal(stats[..., 2].numpy(), ref[..., 2].astype(np.float64))
    return float((err[..., :2] / bound[..., :2]).max())


def intensity_reference(x, stats, coef, normalize, nonzero, channel_wise):
    """fp64 ((x - mean) / sd) a + b from the kernel's statistics, and its bound: the kernel rounds mean and 1 / sd to fp32 (the
    difference those roundings make here is computed, plus u |mean| / sd + u |z| for a mean or variance the device may round
    once differently), then x - m, the product and the fmaf each round once (u each)"""
    n, c = x.shape[:2]
    x = x.reshape(n, c, -1).astype(np.float64)
    a = coef[..., 0].astype(np.float64)[..., None]
    b = coef[..., 1].astype(np.float64)[..., None]
    if not normalize:
        y = x * a + b
        return y, U * np.abs(y) * (1 + 1e-9) + 1e-300
    st = stats.astype(np.float64)
    grp = st if channel_wise else np.repeat(st.sum(1, keepdims=True), c, axis=1)
    k = grp[..., 2]
    mean = np.where(k > 0, grp[..., 0] / np.where(k > 0, k, 1), 0.0)
    var = np.maximum(np.where(k > 0, grp[..., 1] / np.where(k > 0, k, 1) - mean * mean, 0.0), 0.0)
    sd = np.sqrt(var)
    sd = np.where(sd == 0, 1.0, sd)
    mf = mean.astype(np.float32).astype(np.float64)[..., None]
    inv = (1.0 / sd).astype(np.float32).astype(np.float64)[..., None]
    zt = (x - mean[..., None]) / sd[..., None]
    zk = (x - mf) * inv
    ez = np.abs(zk - zt) + 2.01 * U * np.abs(x - mf) * inv + U * (np.abs(mean[..., None]) / sd[..., None] + np.abs(zt))
    skip = (x == 0) if nonzero else np.zeros_like(x, dtype=bool)
    z = np.where(skip, x, zt)
    ez = np.where(skip, 0.0, ez)
    y = z * a + b
    bound = np.abs(a) * ez * (1 + U) + U * (np.abs(y) + np.abs(a) * ez) + 1e-14 * (np.abs(y) + np.abs(b)) + 1e-300
    return y, bound


@pytest.mark.parametrize("case", A.RESAMPLE_CASES, ids=lambda c: c.id)
def test_resample_case(lib, pkg, case):
    sizes, imgs, labs, maps = _resample_data(case)
    y, labels, part, stats, z, coef, ok = _run_resample(lib, pkg, case, sizes, imgs, labs, maps)
    assert ok, "a write outside the output, the labels or the scratch"
    assert not y.isnan().any() and not z.isnan().any()
    worst = 0.0
    for i in range(case.n):
        src = augment_oracle.source_coordinates(torch.tensor(maps[i])[None], case.out)[0]
        ref = geometry_oracle.sample(imgs[i], src, case.padding, "bilinear").numpy()
        srcn = src.numpy()
        for ch in range(case.c):
            bound, delta = resample_bound(imgs[i][ch].double().numpy(), srcn, maps[i], case.padding)
            err = np.abs(y[i, ch].double().numpy() - ref[ch])
            assert (err <= bound).all(), (case.id, i, ch, float((err / bound).max()))
            worst = max(worst, float((err / bound).max()))
        if case.l:
            lref = geometry_oracle.sample(labs[i], src, case.padding, "nearest").numpy()
            tie = _label_ties(srcn, delta, sizes[i], case.padding)
            mism = labels[i].numpy() != lref
            assert not (mism & ~tie[None]).any(), (case.id, i, int((mism & ~tie[None]).sum()))
            assert tie.mean() < 0.05
    wp = _check_partials(y, part, case)
    ws = _check_stats(part, stats, A.resample_geometry(A.vol(case.out))["stats_chain"])
    ref, bound = intensity_reference(y.numpy(), stats.numpy(), coef.numpy(), True, case.nonzero, case.channel_wise)
    err = np.abs(z.reshape(case.n, case.c, -1).double().numpy() - ref)
    assert (err <= bound).all(), (case.id, float((err / bound).max()))
    wi = float((err / bound).max())
    print("%s %s: worst err / bound: resample %.3f, partials %.3f, stats %.3f, intensity %.3f"
          % (case.id, case.key, worst, wp, ws, wi))
    again = _run_resample(lib, pkg, case, sizes, imgs, labs, maps)
    for a_, b_ in zip((y, labels, part, stats, z), again[:5]):
        assert a_ is None or torch.equal(_bits(a_), _bits(b_)), case.id


# ------------------------------------------------------------------------------------------------------------ intensity
def _intensity_data(case):
    g = torch.Generator().manual_seed(sum(map(ord, case.id)))
    S = A.vol(case.dims)
    x = torch.randn(case.n, case.c, S, generator=g) * 2 + 0.5
    if case.nonzero:
        x[torch.rand(x.shape, generator=g) < 0.3] = 0.0
    coef = torch.stack([0.8 + 0.4 * torch.rand(case.n, case.c, generator=g), torch.rand(case.n, case.c, generator=g) - 0.5], -1)
    return x, coef


def _partials(x, nonzero):
    """[n][nb][c][3] fp64 block sums over the restated block ranges (what k_aug_resample leaves for k_aug_stats)"""
    n, c, S = x.shape
    starts = np.array([r[0] for r in A.aug_block_ranges(S)])
    v = x.double().numpy().astype(np.longdouble)
    sel = (v != 0) if nonzero else np.ones_like(v, dtype=bool)
    p = np.stack([np.add.reduceat(v, starts, axis=2), np.add.reduceat(v * v, starts, axis=2),
                  np.add.reduceat(sel.astype(np.longdouble), starts, axis=2)], -1)
    return torch.from_numpy(p.astype(np.float64)).permute(0, 2, 1, 3).contiguous()


def _run_intensity(lib, pkg, case, x, coef):
    n, c, S = x.shape
    nb = A.aug_blocks(S)
    buf, img = _padded(n * c * S, torch.float32, float("nan"), offset=case.offset)
    assert img.data_ptr() % 16 == 4 * case.offset % 16
    img.copy_(x.reshape(-1).to(DEV))
    nbytes = int(lib.b200unet_augment_scratch_bytes(n, c, S))
    sbuf, scratch = _padded(nbytes // 8, torch.float64, float("nan"))
    part = _partials(x, case.nonzero)
    scratch[3 * n * c:].copy_(part.reshape(-1).to(DEV))
    cf = coef.reshape(-1).to(DEV)
    pkg.lib.check(lib.b200unet_augment_intensity(img.data_ptr(), n, c, S, int(case.normalize), int(case.nonzero),
                                                 int(case.channel_wise), cf.data_ptr(), scratch.data_ptr(), pkg.lib.stream_ptr()),
                  "augment_intensity")
    torch.cuda.synchronize()
    ok = _sentinels_intact(buf, img, float("nan"))
    stats = scratch[: 3 * n * c].view(n, c, 3).cpu().clone()
    ok &= not case.normalize or _sentinels_intact(sbuf, scratch, float("nan"))
    return img.view(n, c, S).cpu().clone(), stats, part, ok


@pytest.mark.parametrize("case", A.INTENSITY_CASES, ids=lambda c: c.id)
def test_intensity_case(lib, pkg, case):
    x, coef = _intensity_data(case)
    z, stats, part, ok = _run_intensity(lib, pkg, case, x, coef)
    assert ok, "a write outside the image or the scratch"
    ws = 0.0
    if case.normalize:
        ws = _check_stats(part, stats, A.resample_geometry(A.vol(case.dims))["stats_chain"])
    ref, bound = intensity_reference(x.numpy(), stats.numpy(), coef.numpy(), case.normalize, case.nonzero, case.channel_wise)
    err = np.abs(z.double().numpy() - ref)
    bad = err > bound
    assert not bad.any(), (case.id, np.argwhere(bad)[:5].tolist(), float((err / bound).max()))
    print("%s %s chunks %d: worst err / bound: stats %.3f, intensity %.3f"
          % (case.id, case.key, A.intensity_launch(case.n, case.c, A.vol(case.dims), 4 * case.offset)["chunks"], ws,
             float((err / bound).max())))
    z2, stats2, _, _ = _run_intensity(lib, pkg, case, x, coef)
    assert torch.equal(_bits(z), _bits(z2)) and (not case.normalize or torch.equal(_bits(stats), _bits(stats2)))


# ------------------------------------------------------------------------------------------------------------ foreground
def _mri_like(c, size, seed):
    """zero background, an off-centre N(0, 1) + c core, integer ties in channel 1, a constant channel 2"""
    g = torch.Generator().manual_seed(seed)
    x = torch.zeros((c,) + tuple(size))
    lo = [s // 5 for s in size]
    hi = [max(s - s // 4, l + 1) for s, l in zip(size, lo)]
    core = tuple(slice(a, b) for a, b in zip(lo, hi))
    for ch in range(c):
        shape = tuple(b - a for a, b in zip(lo, hi))
        v = torch.randn(shape, generator=g) + ch
        if ch % 4 == 1:
            v = torch.randint(0, 6, shape, generator=g).float()
        if ch % 4 == 2:
            v = torch.full(shape, 3.5)
        x[(ch,) + core] = v
    return x


def _same_value(a, b):
    """bit for bit, -0 as +0 (numpy's partition leaves either) and every NaN as one value"""
    na, nb = np.isnan(a), np.isnan(b)
    a0 = np.where(na, 0, a + np.float32(0)).astype(np.float32)
    b0 = np.where(nb, 0, b + np.float32(0)).astype(np.float32)
    return bool((na == nb).all() and (a0.view(np.int32) == b0.view(np.int32)).all())


def _run_foreground(lib, pkg, xs, percentile, out, margin, allow_smaller, seed):
    """b200unet_foreground_box on the samples xs (fp32 [C][d][h][w] each, one device buffer); returns host (thr, box, empty,
    affine_out, affine_in, sentinels intact)"""
    n, c = len(xs), xs[0].shape[0]
    sizes = [A.vol(x.shape[1:]) for x in xs]
    offs = np.concatenate([[0], np.cumsum([c * s for s in sizes])])
    flat = torch.empty(int(offs[-1]), dtype=torch.float32)
    for i, x in enumerate(xs):
        flat[offs[i]:offs[i + 1]] = x.reshape(-1)
    dev = flat.to(DEV)
    rows = torch.tensor([[dev.data_ptr() + 4 * int(offs[i]), 0] + list(x.shape[1:]) for i, x in enumerate(xs)], dtype=torch.int64,
                        device=DEV)
    rng = np.random.default_rng(seed)
    ain = np.stack([_rotation_affine(out, rng.uniform(-0.2, 0.2, 3), (0,) if i % 2 else ())[:3].ravel() for i in range(n)])
    ain_d = torch.tensor(ain, dtype=torch.float64, device=DEV)
    ranks = gamma = None
    if percentile is not None:
        idx = [A.percentile_index(s, percentile) for s in sizes]
        ranks = torch.tensor([[lo, hi] * c for lo, hi, _ in idx], dtype=torch.int64, device=DEV)
        gamma = torch.tensor([[float(g)] * c for _, _, g in idx], dtype=torch.float32, device=DEV)
    abuf, aout = _padded(n * 12, torch.float32, float("nan"))
    bbuf, box = _padded(n * 6, torch.int32, -7)
    ebuf, empty = _padded(n, torch.int32, -7)
    tbuf, thr = _padded(n * c, torch.float32, float("nan"))
    nbytes = int(lib.b200unet_foreground_scratch_bytes(n, c))
    assert nbytes > 0
    sbuf, scratch = _padded(nbytes, torch.uint8, 0xCD)
    st = lib.b200unet_foreground_box(rows.data_ptr(), n, c, max(sizes), 1, ranks.data_ptr() if ranks is not None else None,
                                     gamma.data_ptr() if gamma is not None else None, margin, int(allow_smaller), ain_d.data_ptr(),
                                     *out, aout.data_ptr(), box.data_ptr(), empty.data_ptr(),
                                     thr.data_ptr() if ranks is not None else None, scratch.data_ptr(), pkg.lib.stream_ptr())
    pkg.lib.check(st, "foreground_box")
    torch.cuda.synchronize()
    ok = (_sentinels_intact(abuf, aout, float("nan")) and _sentinels_intact(bbuf, box, -7) and _sentinels_intact(ebuf, empty, -7)
          and _sentinels_intact(tbuf, thr, float("nan")) and _sentinels_intact(sbuf, scratch, 0xCD))
    return (thr.cpu().numpy().reshape(n, c).copy(), box.cpu().numpy().reshape(n, 3, 2).copy(), empty.cpu().numpy().copy(),
            aout.cpu().numpy().reshape(n, 3, 4).copy(), ain.reshape(n, 3, 4), ok)


def _check_foreground(xs, res, percentile, out, margin, allow_smaller, name):
    thr, box, empty, aout, ain, ok = res
    assert ok, "a write outside an output or the scratch"
    for i, x in enumerate(xs):
        xn = x.numpy()
        if percentile is not None:
            with np.errstate(invalid="ignore"):
                ref = np.array([np.percentile(xn[ch].reshape(-1), percentile * 100) for ch in range(xn.shape[0])], dtype=np.float32)
            assert _same_value(thr[i], ref), (name, i, thr[i], ref)
        rbox, rempty = geometry_oracle.foreground_box(xn, percentile, margin, allow_smaller)
        assert box[i].tolist() == rbox.tolist() and bool(empty[i]) == rempty, (name, i, box[i].tolist(), rbox.tolist())
        # k_fg_compose: b + s (A p) + (s - 1) / 2 in fp64, rounded to fp32 once
        s = (rbox[:, 1] - rbox[:, 0]) / np.asarray(out, dtype=np.float64)
        want = ain[i] * s[:, None]
        want[:, 3] += rbox[:, 0] + (s - 1) / 2
        assert (np.abs(aout[i] - want) <= U * np.abs(want) * (1 + 1e-9) + 1e-15).all(), (name, i)


@pytest.mark.parametrize("case", A.FOREGROUND_CASES, ids=lambda c: c.id)
def test_foreground_case(lib, pkg, case):
    xs = [_mri_like(case.c, s, 31 * i + len(case.id)) for i, s in enumerate(case.sizes)]
    args = (case.percentile, case.out, case.margin, case.allow_smaller)
    res = _run_foreground(lib, pkg, xs, *args, seed=len(case.id))
    _check_foreground(xs, res, *args, case.id)
    again = _run_foreground(lib, pkg, xs, *args, seed=len(case.id))
    assert all(np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)) for a, b in zip(res[:4], again[:4]))
    print("%s %s: %d samples, thresholds, boxes and empty flags exact" % (case.id, case.keys, len(xs)))


@pytest.mark.parametrize("case", A.SELECT_CASES, ids=lambda c: c.id)
def test_select_case(lib, pkg, case):
    x = torch.from_numpy(case.build()).view(1, case.n, 1, 1)
    args = (case.percentile, (4, 4, 4), 1, True)
    res = _run_foreground(lib, pkg, [x], *args, seed=1)
    _check_foreground([x], res, *args, case.id)
    again = _run_foreground(lib, pkg, [x], *args, seed=1)
    assert np.array_equal(res[0].view(np.uint32), again[0].view(np.uint32))
    print("%s (diverges at pass %s): thr %r bit for bit" % (case.id, case.tagged, float(res[0][0, 0])))


def test_too_many_planes_are_refused_before_a_launch(lib, pkg):
    """n * c > 65535 planes: the size query returns 0 naming n and c, and the launch returns E_UNSUPPORTED without touching
    its buffers (real, too small ones here)"""
    assert lib.b200unet_foreground_scratch_bytes(4097, 16) == 0
    assert "n=4097" in lib.b200unet_last_error().decode()
    buf = torch.full((64,), 7, dtype=torch.int64, device=DEV)
    p = buf.data_ptr()
    st = lib.b200unet_foreground_box(p, 4097, 16, 1000, 1, p, p, 1, 1, p, 8, 8, 8, p, p, p, p, p, pkg.lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == -2 and "c=16" in lib.b200unet_last_error().decode()
    assert (buf == 7).all()
