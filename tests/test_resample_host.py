"""Host side of the resample onto the image file's grid (``prepost.resample_to_match``, ``volumetric_predictions(resample=True)``):
the index map composed from the metadata affines against numpy, the metadata forms a loader may hand over, the errors, and a
marshalling dry run of ``b200unet_resample_to_grid`` against a stub of the library.  The kernel's values are checked in
tests/test_gpu_resample.py."""
import contextlib
import os
import sys

import numpy as np
import pytest
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import resample_cases as rc  # noqa: E402

ENTRY = "b200unet_resample_to_grid"


# ------------------------------------------------------------------------------------------------ index map
def _map(a_pred, a_file, pkg):
    """target = the file's grid, source = the prediction's grid"""
    return pkg.prepost.index_map(a_pred, a_file)


def test_index_map_of_a_crop_is_an_integer_shift(pkg):
    a0 = rc.file_affine((0.9375, 0.9375, 1.4), origin=(-120.3, 97.1, 12.0))
    m = _map(a0 @ rc.crop((30, 25, 10)), a0, pkg)
    want = np.hstack([np.eye(3), [[-30.0], [-25.0], [-10.0]]])
    assert np.array_equal(m, want)                     # snapped: the inexact spacing leaves no 1e-15 fraction


def test_index_map_of_a_resize_is_the_inverse_scale(pkg):
    a0 = rc.file_affine((0.7, 0.7, 1.2))
    m = _map(a0 @ rc.resize((144, 216, 224), (192, 192, 192)), a0, pkg)
    s = np.array([192 / 144, 192 / 216, 192 / 224])
    want = np.hstack([np.diag(s), ((s - 1) / 2)[:, None]])                  # new = (old + 0.5) * new / old - 0.5
    np.testing.assert_allclose(m, want, rtol=0, atol=1e-13)
    # the centre of the first and last old voxels
    for old in ((0, 0, 0), (143, 215, 223)):
        new = (np.asarray(old) + 0.5) * 192 / np.array([144, 216, 224]) - 0.5
        np.testing.assert_allclose(m @ np.r_[old, 1.0], new, atol=1e-12)


def test_index_map_of_lps_to_ras_is_a_flip_and_a_permutation(pkg):
    shape = (40, 50, 30)
    a0 = rc.file_affine((0.8, 0.8, 2.5), origin=(10.0, -4.0, 7.0), lps=True)
    p, oshape = rc.flip_perm(shape, perm=(2, 0, 1), flips=(1, 2))
    m = _map(a0 @ p, a0, pkg)
    assert oshape == (30, 40, 50)
    for v in ((0, 0, 0), (39, 49, 29), (7, 11, 13)):
        # file voxel v lies at oriented index (v[2], 39 - v[0], 49 - v[1])
        assert np.array_equal(m @ np.r_[v, 1.0], np.array([v[2], 39 - v[0], 49 - v[1]], dtype=np.float64))


@pytest.mark.parametrize("name", sorted(rc.GRIDS))
def test_index_map_of_orientation_crop_and_resize_composes(pkg, name):
    a0, shape, a, pshape = rc.grid(name)
    m = _map(a, a0, pkg)
    np.testing.assert_allclose(m, rc.expected_index_map(name), rtol=0, atol=1e-12)
    # the file's corner voxels: inside the prediction grid, or beyond its edge only where the crop cut the volume
    c = rc.target_coords(m, shape)
    assert c.min() < -0.5 and (c.max(axis=(1, 2, 3)) > np.asarray(pshape) - 0.5).all()


def test_index_map_identity_and_tolerance(pkg):
    a0 = rc.file_affine((1.1, 0.9, 3.0), origin=(1.0, 2.0, 3.0))
    assert np.array_equal(pkg.prepost.index_map(a0, a0), np.eye(4)[:3])
    near = a0.copy()
    near[0, 3] += 1e-7                                # fp32-stored metadata: well inside INDEX_MAP_TOL of a voxel
    assert np.array_equal(pkg.prepost.index_map(near, a0), np.eye(4)[:3])
    far = a0.copy()
    far[0, 3] += 1e-3
    assert not np.array_equal(pkg.prepost.index_map(far, a0), np.eye(4)[:3])


# ------------------------------------------------------------------------------------------------ errors
def test_unsupported_modes_raise_not_implemented(pkg):
    x = torch.zeros(1, 4, 4, 4)
    for mode in ("bicubic", "area", 3, 1, None):
        with pytest.raises(NotImplementedError):
            pkg.prepost.resample_to_match(x, np.eye(4), np.eye(4), (4, 4, 4), mode=mode)
    assert [pkg.prepost.resample_mode(m) for m in ("trilinear", "bilinear", "linear", "nearest")] == [0, 0, 0, 1]


def test_cpu_tensor_raises_no_cpu_fallback(pkg):
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pkg.prepost.resample_to_match(torch.zeros(1, 4, 4, 4), np.eye(4), np.eye(4), (5, 5, 5))


class _Meta(torch.Tensor):
    pass


class _FakeCudaMeta(torch.Tensor):
    """a CPU tensor with ``meta`` that claims to live on a CUDA device (only the host layer's entry checks read the flag)"""
    is_cuda = True


def _item(cls=_Meta, n=2, shape=(6, 7, 5), **meta):
    x = torch.rand((n, 1) + shape, generator=torch.Generator().manual_seed(0)).as_subclass(cls)
    x.meta = dict(filename_or_obj=["f%d.nii.gz" % i for i in range(n)], **meta)
    return x


def test_missing_metadata_key_names_the_key_and_the_loader(pkg):
    model = nn.Conv3d(1, 1, 1)
    full = dict(affine=torch.eye(4)[None].repeat(2, 1, 1), original_affine=np.stack([np.eye(4)] * 2),
                spatial_shape=torch.tensor([[6, 7, 5]] * 2))
    for key in ("affine", "original_affine", "spatial_shape"):
        meta = {k: v for k, v in full.items() if k != key}
        with pytest.raises(KeyError, match=r"%s.*LoadImageD" % key):
            pkg.predict.volumetric_predictions(model, [{"image": _item(**meta)}], "out", resample=True)
    with pytest.raises(NotImplementedError):
        pkg.predict.volumetric_predictions(model, [{"image": _item(**full)}], "out", resample=True, interpolation="bicubic")
    # resample=False reads none of them
    res = pkg.predict.volumetric_predictions(model, [{"image": _item()}], "out", interpolation="bicubic")
    assert [tuple(r[1].shape) for r in res] == [(1, 6, 7, 5)] * 2


# ------------------------------------------------------------------------------------------------ marshalling dry run
@pytest.fixture()
def stubbed(pkg, monkeypatch):
    """the library with ``b200unet_resample_to_grid`` replaced by a check of the argument count and ctypes convertibility
    against the binding's signature; records the arguments of each call"""
    L = pkg.lib
    real = L.load_library()
    res, argtypes = L._SIGS[ENTRY]
    calls = []

    class Stub:
        def __getattr__(self, name):
            return getattr(real, name)

    def f(*args):
        assert len(args) == len(argtypes), "%s: %d arguments, signature has %d" % (ENTRY, len(args), len(argtypes))
        for i, (v, t) in enumerate(zip(args, argtypes)):
            try:
                t.from_param(v)
            except Exception as e:  # noqa: BLE001
                raise AssertionError("%s: argument %d (%r) does not convert to %s: %s" % (ENTRY, i, v, t, e))
        calls.append(dict(c=args[1], src=tuple(args[2:5]), affine=np.array(args[5][:12]), mode=args[6], dst=tuple(args[8:11])))
        return 0

    stub = Stub()
    stub.b200unet_resample_to_grid = f
    monkeypatch.setattr(L, "_lib", stub)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    monkeypatch.setattr(torch.cuda, "device", lambda *_a, **_k: contextlib.nullcontext())
    return calls


def _fake(t):
    return t.as_subclass(_FakeCudaMeta)


def test_resample_to_match_marshals_one_call_per_item(pkg, stubbed):
    a0, shape, a, pshape = rc.grid("brats")
    x = _fake(torch.rand((3,) + pshape[:1] + (4, 4)))       # [C, D, H, W]; the map does not depend on the source extents
    y = pkg.prepost.resample_to_match(x, a, a0, shape)
    assert y.shape == (3,) + shape and y.dtype == torch.float32
    assert len(stubbed) == 1 and stubbed[0]["c"] == 3 and stubbed[0]["src"] == (128, 4, 4) and stubbed[0]["dst"] == shape
    assert stubbed[0]["mode"] == 0 and np.array_equal(stubbed[0]["affine"], pkg.prepost.index_map(a, a0).ravel())
    # a batch with one affine per item, nearest
    xb = _fake(torch.rand(2, 104, 5, 6, 7))
    yb = pkg.prepost.resample_to_match(xb, torch.tensor(np.stack([a, a0])), a0, torch.tensor([9, 8, 7]), mode="nearest")
    assert yb.shape == (2, 104, 9, 8, 7) and [c["mode"] for c in stubbed[1:]] == [1, 1]
    assert np.array_equal(stubbed[2]["affine"], np.eye(4)[:3].ravel())
    with pytest.raises(ValueError):
        pkg.prepost.resample_to_match(xb, np.stack([a, a0, a]), a0, (9, 8, 7))
    with pytest.raises(ValueError):
        pkg.prepost.resample_to_match(xb, a, a0, (9, 8))


def test_identical_grids_copy_without_a_kernel(pkg, stubbed):
    a0 = rc.file_affine((0.9, 0.9, 1.3))
    x = torch.randn(2, 5, 6, 7)
    x[0, 1, 2, 3] = float("nan")
    y = pkg.prepost.resample_to_match(_fake(x), a0, a0.astype(np.float32), (5, 6, 7))
    assert not stubbed and type(y) is torch.Tensor
    assert torch.equal(y.view(torch.int32), x.view(torch.int32))
    pkg.prepost.resample_to_match(_fake(x), a0, a0, (5, 6, 8))               # same affine, other shape: resampled
    assert len(stubbed) == 1


@pytest.mark.parametrize("form", ["batched", "per_item", "numpy_batched", "shared"])
def test_volumetric_predictions_reads_each_metadata_form(pkg, stubbed, form):
    """the prediction of item i goes from meta["affine"][i] to (meta["original_affine"][i], meta["spatial_shape"][i])"""
    a0, shape, a, _ = rc.grid("brats")
    a1 = a0.copy()
    a1[:3, 3] += (2.0, -1.0, 0.5)
    pred_aff, file_aff, shapes = [a, a @ rc.crop((1, 2, 3))], [a0, a1], [shape, (200, 210, 90)]
    if form == "batched":                          # as the collate function leaves them
        meta = dict(affine=torch.tensor(np.stack(pred_aff)), original_affine=torch.tensor(np.stack(file_aff)),
                    spatial_shape=torch.tensor(shapes))
    elif form == "per_item":
        meta = dict(affine=[torch.tensor(v) for v in pred_aff], original_affine=list(file_aff), spatial_shape=[tuple(s) for s in shapes])
    elif form == "numpy_batched":
        meta = dict(affine=np.stack(pred_aff), original_affine=np.stack(file_aff), spatial_shape=np.array(shapes))
    else:                                          # one grid for the whole batch
        pred_aff, file_aff, shapes = [a, a], [a0, a0], [shape, shape]
        meta = dict(affine=torch.tensor(a), original_affine=a0, spatial_shape=shape)
    model = nn.Conv3d(1, 2, 1)
    x = _item(_FakeCudaMeta, **meta)
    written = []
    res = pkg.predict.volumetric_predictions(model, [{"image": x}], "out", activation="sigmoid", resample=True,
                                             writer=lambda fn, t, d: written.append((fn, tuple(t.shape))))
    assert [tuple(r[1].shape) for r in res] == [(2,) + tuple(s) for s in shapes]
    assert written == [("f%d.nii.gz" % i, (2,) + tuple(s)) for i, s in enumerate(shapes)]
    assert len(stubbed) == 2
    for i, call in enumerate(stubbed):
        assert call["c"] == 2 and call["src"] == (6, 7, 5) and call["dst"] == tuple(shapes[i]) and call["mode"] == 0
        assert np.array_equal(call["affine"], pkg.prepost.index_map(pred_aff[i], file_aff[i]).ravel())
