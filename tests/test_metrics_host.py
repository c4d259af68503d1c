"""Boundary-distance metrics without a GPU: the MONAI restatement (tests/metrics_oracle.py) against brute-force nearest-edge
loops, argument validation, prepare_spacing and the aggregate reductions."""
import numpy as np
import pytest
import torch

import metrics_oracle as orc


@pytest.fixture(scope="module")
def M(pkg):
    return pkg.metrics


def _cases():
    rng = np.random.default_rng(0)
    shape = (5, 6, 7)
    blob = np.zeros(shape, bool); blob[1:4, 2:5, 1:6] = True
    blob2 = np.zeros(shape, bool); blob2[2:5, 0:3, 3:7] = True
    faces = np.zeros(shape, bool); faces[0] = True; faces[:, -1] = True; faces[..., 0] = True
    full = np.ones(shape, bool)
    one = np.zeros(shape, bool); one[2, 3, 4] = True
    one2 = np.zeros(shape, bool); one2[4, 0, 6] = True
    empty = np.zeros(shape, bool)
    return {
        "blobs": (blob, blob2), "random": (rng.random(shape) < 0.4, rng.random(shape) < 0.3), "faces": (faces, blob),
        "full": (full, one), "singles": (one, one2), "pred_empty": (empty, blob), "gt_empty": (blob, empty),
        "both_empty": (empty, empty), "extent1": (rng.random((1, 6, 7)) < 0.5, rng.random((1, 6, 7)) < 0.5),
        "odd": (rng.random((3, 5, 9)) < 0.3, rng.random((3, 5, 9)) < 0.6),
    }


@pytest.mark.parametrize("name", list(_cases()))
@pytest.mark.parametrize("spacing", [(1.0, 1.0, 1.0), (1.0, 0.8, 2.5)])
def test_oracle_matches_brute_force(name, spacing):
    p, g = _cases()[name]
    got = orc.pair_distances(p, g, spacing)
    ref = orc.brute_force_distances(p, g, spacing)
    for a, b in zip(got, ref):
        assert a.shape == b.shape
        if spacing == (1.0, 1.0, 1.0):
            assert np.array_equal(a, b)
        else:
            assert np.all((a == b) | (np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32)) <= 1))


def test_oracle_empty_mask_table():
    c = _cases()
    p = np.stack([c["pred_empty"][0], c["gt_empty"][0], c["both_empty"][0]])[None]
    g = np.stack([c["pred_empty"][1], c["gt_empty"][1], c["both_empty"][1]])[None]
    for pct in (None, 95):
        hd = orc.hausdorff(p, g, True, pct)[0]
        assert np.isinf(hd[0]) and np.isinf(hd[1]) and np.isnan(hd[2])
    asd = orc.average_surface(p, g, True, True)[0]
    assert np.isinf(asd[0]) and np.isinf(asd[1]) and np.isnan(asd[2])
    nsd = orc.surface_dice(p, g, [1.0] * 3, True)[0]
    assert nsd[0] == 0 and nsd[1] == 0 and np.isnan(nsd[2])


def test_oracle_foreground_is_value_one():
    x = np.array([0, 1, 2, 0.7, 1.0], np.float32)
    assert orc.foreground(x).tolist() == [False, True, False, False, True]


def test_prepare_spacing_forms(M):
    assert M.prepare_spacing(None, 2, 3) == [None, None]
    assert M.prepare_spacing(1.5, 3, 3) == [1.5] * 3
    assert M.prepare_spacing((1.0, 0.8, 2.5), 2, 3) == [(1.0, 0.8, 2.5)] * 2
    assert M.prepare_spacing([[1, 2, 3], [4, 5, 6]], 2, 3) == [[1, 2, 3], [4, 5, 6]]
    for bad in ([[1, 2, 3]], (1.0, 2.0), [[1, 2], [3, 4]], [1, 2.0, 3], ["a", "b", "c"], [[1, 2, "x"], [1, 2, 3]]):
        with pytest.raises(ValueError):
            M.prepare_spacing(bad, 2, 3)
    np.testing.assert_array_equal(M._spacing_rows(None, 2), np.ones((2, 3)))
    np.testing.assert_array_equal(M._spacing_rows(2, 1), np.full((1, 3), 2.0))
    np.testing.assert_array_equal(M._spacing_rows([(1, 2, 3), (4, 5, 6)], 2), [[1, 2, 3], [4, 5, 6]])


def test_argument_errors(M, pkg):
    x = torch.zeros((1, 2, 4, 4, 4), dtype=torch.bool)
    with pytest.raises(NotImplementedError):
        M.compute_hausdorff_distance(x, x, distance_metric="chessboard")
    with pytest.raises(NotImplementedError):
        M.compute_average_surface_distance(x, x, distance_metric="taxicab")
    with pytest.raises(NotImplementedError):
        M.compute_surface_dice(x, x, [1.0], use_subvoxels=True)
    with pytest.raises(NotImplementedError):
        M.compute_hausdorff_distance(x[..., 0], x[..., 0])                    # 2-D images
    with pytest.raises(NotImplementedError):
        pkg.SurfaceDiceMetric([1.0], use_subvoxels=True)
    for pct in (-1, 100.5, 250):
        with pytest.raises(ValueError):
            M.compute_hausdorff_distance(x, x, percentile=pct)
        with pytest.raises(ValueError):
            pkg.HausdorffDistanceMetric(percentile=pct)
    with pytest.raises(ValueError):
        M.compute_hausdorff_distance(x, x[:, :, :3])                           # shapes differ
    with pytest.raises(ValueError):
        M.compute_surface_dice(x, x, [1.0, 2.0])                               # C' = 1 after dropping the background
    with pytest.raises(ValueError):
        M.compute_hausdorff_distance(x, x, spacing=(1.0, 2.0))                 # malformed spacing
    with pytest.raises(ValueError):
        M.compute_hausdorff_distance(x, x, spacing=[(1, 1, 1), (1, 1, 1)])     # B = 1
    with pytest.raises(TypeError):
        M.compute_hausdorff_distance(x.long(), x.long())
    with pytest.raises(RuntimeError, match="CUDA"):                            # no CPU fallback
        M.compute_hausdorff_distance(x, x)
    with pytest.raises(RuntimeError, match="CUDA"):
        M.compute_surface_dice([x[0]], [x[0]], [1.0])


def test_percentile_zero_and_none_take_the_max(M):
    assert M._quantile(None) == 0.0 and M._quantile(0) == 0.0
    assert M._quantile(95) == float(np.float32(0.95)) and M._quantile(100) == 1.0


def test_aggregate_reductions(M, pkg):
    nan, inf = float("nan"), float("inf")
    f = torch.tensor([[1.0, nan, 3.0], [nan, nan, 5.0], [2.0, 4.0, inf]])
    m = pkg.HausdorffDistanceMetric(get_not_nans=True)
    m._buffer = [f[:2], f[2:]]
    assert torch.equal(m.get_buffer(), f) or torch.allclose(m.get_buffer(), f, equal_nan=True)
    expect = {
        "mean": (torch.tensor([inf]), torch.tensor(3.0)),          # shape [1], as MONAI returns it
        "sum": (torch.tensor(inf), torch.tensor(6.0)),
        "mean_batch": (torch.tensor([1.5, 4.0, inf]), torch.tensor([2.0, 1.0, 3.0])),
        "sum_batch": (torch.tensor([3.0, 4.0, inf]), torch.tensor([2.0, 1.0, 3.0])),
        "mean_channel": (torch.tensor([2.0, 5.0, inf]), torch.tensor([2.0, 1.0, 3.0])),
        "sum_channel": (torch.tensor([4.0, 5.0, inf]), torch.tensor([2.0, 1.0, 3.0])),
    }
    for red, (ef, en) in expect.items():
        got, nn = m.aggregate(red)
        assert torch.equal(got, ef), red
        assert torch.equal(nn, en), red
    got, nn = m.aggregate("none")
    assert torch.allclose(got, f, equal_nan=True) and torch.equal(nn, (~torch.isnan(f)).float())
    finite = torch.tensor([[1.0, nan], [3.0, 5.0]])
    m2 = pkg.SurfaceDistanceMetric()
    m2._buffer = [finite]
    assert torch.allclose(m2.aggregate(), torch.tensor((1.0 + 4.0) / 2))     # channel means 1 and 4, then the batch
    assert torch.equal(m2.aggregate("mean_batch"), torch.tensor([2.0, 5.0]))
    all_nan = pkg.SurfaceDiceMetric([1.0])
    all_nan._buffer = [torch.full((2, 2), nan)]
    assert all_nan.aggregate().item() == 0.0
    assert torch.isnan(f).sum() == 3                                          # the buffer is not modified
    with pytest.raises(ValueError):
        m.aggregate("median")
    with pytest.raises(ValueError):
        pkg.HausdorffDistanceMetric().aggregate()                             # nothing buffered
