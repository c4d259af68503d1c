"""HD / HD95, average surface distance and surface Dice on the device against the scipy restatement of MONAI
(tests/metrics_oracle.py): exact with unit spacing (nan and inf included), 1 fp32 ulp with anisotropic spacing, ASD within 1e-6
of the oracle's fp64 mean; bit-identical run to run."""
import numpy as np
import pytest
import torch

import metrics_oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M(pkg):
    return pkg.metrics


def blobs(rng, shape, n, rmin, rmax):
    """n random ellipsoids per volume (lesion-like), bool [*shape]"""
    D, H, W = shape
    z, y, x = np.ogrid[:D, :H, :W]
    m = np.zeros(shape, bool)
    for _ in range(n):
        c = [rng.uniform(0, s) for s in shape]
        r = [rng.uniform(rmin, rmax) for _ in range(3)]
        m |= ((z - c[0]) / r[0]) ** 2 + ((y - c[1]) / r[1]) ** 2 + ((x - c[2]) / r[2]) ** 2 <= 1
    return m


def batch(rng, b, c, shape, n=3, rmin=2, rmax=8):
    p = np.stack([np.stack([blobs(rng, shape, n, rmin, rmax) for _ in range(c)]) for _ in range(b)])
    g = np.stack([np.stack([blobs(rng, shape, n, rmin, rmax) for _ in range(c)]) for _ in range(b)])
    return p, g


def cuda(x, dtype=torch.bool):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dtype).cuda()


def ulp_equal(a, b, ulps=1):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    fin = np.isfinite(a) & np.isfinite(b)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    return bool(np.all(same | (fin & (np.abs(ia - ib) <= ulps))))


def exact(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def asd_close(gpu, ref):
    g, r = np.asarray(gpu, np.float64), np.asarray(ref, np.float64)
    same = (g == r) | (np.isnan(g) & np.isnan(r))
    fin = np.isfinite(g) & np.isfinite(r)
    close = np.abs(np.where(fin, g, 0) - np.where(fin, r, 0)) <= 1e-6 * np.abs(np.where(fin, r, 0))
    return bool(np.all(same | (fin & close)))


def check_all(M, p, g, spacing=None, include_background=True, thr=(1.0, 2.0, 0.5), exact_ok=True):
    c = p.shape[1] if include_background or p.shape[1] == 1 else p.shape[1] - 1
    th = [thr[i % len(thr)] for i in range(c)]
    cmp = exact if exact_ok else ulp_equal
    for pct in (None, 0, 50, 95, 100):
        for directed in (False, True):
            got = M.compute_hausdorff_distance(cuda(p), cuda(g), include_background, percentile=pct, directed=directed,
                                               spacing=spacing).cpu().numpy()
            ref = orc.hausdorff(p, g, include_background, pct, directed, spacing)
            assert cmp(got, ref), (pct, directed, got, ref)
    for sym in (False, True):
        got = M.compute_average_surface_distance(cuda(p), cuda(g), include_background, sym, spacing=spacing).cpu().numpy()
        assert asd_close(got, orc.average_surface(p, g, include_background, sym, spacing)), sym
    got = M.compute_surface_dice(cuda(p), cuda(g), th, include_background, spacing=spacing).cpu().numpy()
    assert cmp(got, orc.surface_dice(p, g, th, include_background, spacing)), (got, orc.surface_dice(p, g, th, include_background,
                                                                                                     spacing))


def test_blobs_small_all_options(M):
    rng = np.random.default_rng(0)
    p, g = batch(rng, 2, 3, (24, 28, 33))
    check_all(M, p, g, include_background=True)
    check_all(M, p, g, include_background=False)


def test_anisotropic_and_per_item_spacing(M):
    rng = np.random.default_rng(1)
    p, g = batch(rng, 2, 2, (20, 31, 26))
    check_all(M, p, g, spacing=(1.0, 0.8, 2.5), exact_ok=False)
    check_all(M, p, g, spacing=[(1.0, 0.8, 2.5), (0.7, 1.3, 1.1)], exact_ok=False)
    check_all(M, p, g, spacing=2.0)


def test_special_masks(M):
    """faces, full volume, single voxels, one mask empty (each side), both empty, in one batch"""
    shape = (9, 10, 11)
    faces = np.zeros(shape, bool); faces[:, :, :2] = True; faces[0] = True; faces[:, -1] = True
    full = np.ones(shape, bool)
    one = np.zeros(shape, bool); one[4, 5, 6] = True
    one2 = np.zeros(shape, bool); one2[0, 0, 0] = True
    empty = np.zeros(shape, bool)
    cases = [(faces, full), (full, one), (one, one2), (one, empty), (empty, faces), (empty, empty), (full, full)]
    p = np.stack([c[0] for c in cases])[None]
    g = np.stack([c[1] for c in cases])[None]
    check_all(M, p, g, include_background=True)
    hd = M.compute_hausdorff_distance(cuda(p), cuda(g), True, percentile=95).cpu().numpy()[0]
    assert np.isinf(hd[3]) and np.isinf(hd[4]) and np.isnan(hd[5]) and hd[6] == 0
    nsd = M.compute_surface_dice(cuda(p), cuda(g), [1.0] * 7, True).cpu().numpy()[0]
    assert nsd[3] == 0 and nsd[4] == 0 and np.isnan(nsd[5]) and nsd[6] == 1


@pytest.mark.parametrize("shape", [(37, 64, 129), (1, 40, 50), (30, 1, 45), (25, 33, 1), (256, 3, 5)])
def test_odd_extents(M, shape):
    rng = np.random.default_rng(sum(shape))
    p, g = batch(rng, 1, 2, shape, n=4, rmin=1, rmax=12)
    check_all(M, p, g, include_background=True)


def test_dtypes_values_strides_and_lists(M):
    rng = np.random.default_rng(3)
    p, g = batch(rng, 2, 3, (16, 20, 24))
    ref = orc.hausdorff(p, g, False, 95)
    # fp32 with values other than 0 and 1: only exact 1.0 is foreground
    pf = torch.from_numpy(p.astype(np.float32)).cuda()
    pf = torch.where(pf == 0, torch.full_like(pf, 0.7), pf)
    gu = cuda(g, torch.uint8) * 1
    gu[gu == 0] = 2
    assert exact(M.compute_hausdorff_distance(pf, gu, percentile=95).cpu().numpy(), ref)
    # non-contiguous: a channels-last copy and a strided slice of a wider batch
    pn = cuda(p, torch.uint8).permute(0, 1, 4, 3, 2).contiguous().permute(0, 1, 4, 3, 2)
    wide = torch.zeros((2, 3, 16, 20, 48), dtype=torch.bool, device="cuda")
    wide[..., ::2] = cuda(g)
    gn = wide[..., ::2]
    assert not pn.is_contiguous() and not gn.is_contiguous()
    assert exact(M.compute_hausdorff_distance(pn, gn, percentile=95).cpu().numpy(), ref)
    # lists of [C, D, H, W]
    got = M.compute_hausdorff_distance([cuda(x) for x in p], [cuda(x) for x in g], percentile=95).cpu().numpy()
    assert exact(got, ref)


def test_cumulative_classes(M, pkg):
    rng = np.random.default_rng(4)
    p, g = batch(rng, 2, 3, (18, 22, 20))
    p2, g2 = batch(rng, 1, 3, (18, 22, 20))
    hd = pkg.HausdorffDistanceMetric(percentile=95, reduction="mean_batch", get_not_nans=True)
    asd = pkg.SurfaceDistanceMetric(symmetric=True)
    nsd = pkg.SurfaceDiceMetric([1.0, 1.5])
    for a, b in ((p, g), (p2, g2)):
        hd(cuda(a), cuda(b))
        asd(cuda(a), cuda(b), spacing=(1.0, 0.8, 2.5))
        nsd([cuda(x) for x in a], [cuda(x) for x in b])
    P, G = np.concatenate([p, p2]), np.concatenate([g, g2])
    assert exact(hd.get_buffer().cpu().numpy(), orc.hausdorff(P, G, False, 95))
    f, nn = hd.aggregate()
    ref, _ = M.do_metric_reduction(torch.from_numpy(orc.hausdorff(P, G, False, 95)), "mean_batch")
    assert torch.equal(f.cpu(), ref)
    assert asd_close(asd.get_buffer().cpu().numpy(), orc.average_surface(P, G, False, True, (1.0, 0.8, 2.5)))
    assert exact(nsd.get_buffer().cpu().numpy(), orc.surface_dice(P, G, [1.0, 1.5]))
    nsd.reset()
    assert nsd.get_buffer() is None


def test_combined_call_matches_separate_calls(M):
    rng = np.random.default_rng(5)
    p, g = batch(rng, 2, 2, (20, 24, 28))
    P, G = cuda(p), cuda(g)
    out = M.compute_surface_metrics(P, G, True, percentile=95, class_thresholds=[1.0, 2.0])
    assert torch.equal(out["hd"], M.compute_hausdorff_distance(P, G, True, percentile=95))
    assert torch.equal(out["asd"], M.compute_average_surface_distance(P, G, True))
    assert torch.equal(out["nsd"], M.compute_surface_dice(P, G, [1.0, 2.0], True))


def test_deterministic(M):
    rng = np.random.default_rng(6)
    p, g = batch(rng, 2, 3, (40, 48, 56), n=5, rmin=2, rmax=14)
    P, G = cuda(p), cuda(g)
    a = [M.compute_surface_metrics(P, G, True, percentile=95, symmetric=True, class_thresholds=[1, 2, 3], spacing=(1.0, 0.8, 2.5))
         for _ in range(2)]
    for k in a[0]:
        assert torch.equal(a[0][k], a[1][k]), k


def test_brats_size(M):
    """240 x 240 x 155, B = 2, C = 3 with lesion-like blobs: HD95 exact, one launch sequence for the whole batch"""
    rng = np.random.default_rng(7)
    shape = (240, 240, 155)
    p, g = batch(rng, 2, 3, shape, n=3, rmin=4, rmax=30)
    P, G = cuda(p), cuda(g)
    got = M.compute_hausdorff_distance(P, G, include_background=True, percentile=95).cpu().numpy()
    assert exact(got, orc.hausdorff(p, g, True, 95))
    got_asd = M.compute_average_surface_distance(P, G, include_background=True, symmetric=True).cpu().numpy()
    assert asd_close(got_asd, orc.average_surface(p, g, True, True))


def test_256_cube_accepted_and_257_rejected(M):
    P = torch.zeros((2, 3, 256, 256, 256), dtype=torch.bool, device="cuda")
    P[:, :, 100:120, 50:90, 30:31] = True
    G = torch.zeros_like(P)
    G[:, :, 10:12, 200:230, 240:256] = True
    got = M.compute_hausdorff_distance(P, G, include_background=True).cpu().numpy()
    ref = orc.hausdorff(P[:1, :1].cpu().numpy(), G[:1, :1].cpu().numpy(), True)
    assert np.all(got == ref[0, 0])
    with pytest.raises(RuntimeError, match="at most 256"):
        M.compute_hausdorff_distance(torch.zeros((1, 1, 257, 4, 4), dtype=torch.bool, device="cuda"),
                                     torch.zeros((1, 1, 257, 4, 4), dtype=torch.bool, device="cuda"))
