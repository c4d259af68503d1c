"""Resample onto the image file's grid (``prepost.resample_to_match``, ``csrc/resample.cu``) against fp64 oracles
(tests/resample_cases.py): trilinear with border padding against scipy's map_coordinates(order=1, mode="nearest"), nearest
against an explicit round half to even; exact copies for flips, permutations, integer shifts and identical grids; and
``volumetric_predictions(resample=True)`` end to end."""
import os
import sys

import numpy as np
import pytest
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import resample_cases as rc  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _probs(shape, seed=0):
    return torch.rand(shape, generator=torch.Generator().manual_seed(seed))


def _scaled(src_shape, dst_shape, angle=0.0, shear=0.0, offset=(0.0, 0.0, 0.0)):
    """(prediction affine, file affine) whose index map scales the file's extents onto the prediction's, optionally rotated
    about the volume centre and sheared"""
    a_file = rc.file_affine((1.0, 1.0, 1.0))
    s = np.asarray(src_shape, dtype=np.float64) / np.asarray(dst_shape, dtype=np.float64)
    c, sn = np.cos(angle), np.sin(angle)
    lin = np.array([[c, -sn, shear], [sn, c, 0.0], [0.0, shear, 1.0]]) @ np.diag(s)
    ctr_dst = (np.asarray(dst_shape) - 1) / 2
    ctr_src = (np.asarray(src_shape) - 1) / 2
    m = np.eye(4)
    m[:3, :3] = lin
    m[:3, 3] = ctr_src - lin @ ctr_dst + np.asarray(offset)
    return a_file @ np.linalg.inv(m), a_file          # index_map(a_pred, a_file) = m


def _check(pkg, x, a_pred, a_file, dst_shape, mode="trilinear", tol=1e-6):
    got = pkg.prepost.resample_to_match(x.to(DEV), a_pred, a_file, dst_shape, mode=mode)
    m = pkg.prepost.index_map(a_pred, a_file)
    ref = rc.oracle(x.double().numpy(), m, dst_shape, mode)
    assert got.shape == (x.shape[0],) + tuple(dst_shape) and got.dtype == torch.float32
    err = float(np.abs(got.cpu().double().numpy() - ref).max())
    print("resample %s -> %s C=%d %s: max abs %.3e" % (tuple(x.shape[1:]), tuple(dst_shape), x.shape[0], mode, err))
    if mode == "nearest":
        assert err == 0.0
    else:
        assert err <= tol
    return got


@pytest.mark.parametrize("c,src,dst,angle,shear", [
    (3, (20, 24, 16), (37, 29, 41), 0.0, 0.0),          # upsampling, anisotropic extents
    (1, (48, 40, 36), (23, 31, 17), 0.0, 0.0),          # downsampling
    (104, (12, 14, 10), (16, 13, 11), 0.4, 0.15),       # rotated and sheared, the widest head
    (1, (30, 26, 22), (33, 35, 21), 0.25, 0.1),
])
def test_trilinear_matches_map_coordinates(pkg, c, src, dst, angle, shear):
    a_pred, a_file = _scaled(src, dst, angle, shear, offset=(0.3, -1.7, 0.6))
    _check(pkg, _probs((c,) + src, seed=c), a_pred, a_file, dst)


@pytest.mark.parametrize("name", sorted(rc.GRIDS))
def test_dataset_grids_match_map_coordinates(pkg, name):
    """the BraTS grid (128^3 -> 240 x 240 x 155, C = 3) and the SPPIN grid (192^3 -> 256 x 256 x 160, oblique affine)"""
    a0, shape, a, pshape = rc.grid(name)
    c = 3 if name == "brats" else 1
    _check(pkg, _probs((c,) + pshape, seed=1), a, a0, shape)


@pytest.mark.parametrize("c,src,dst,angle", [(3, (20, 24, 16), (41, 47, 31), 0.0), (1, (40, 36, 30), (20, 18, 15), 0.0),
                                             (104, (12, 14, 10), (16, 13, 11), 0.35)])
def test_nearest_is_exact(pkg, c, src, dst, angle):
    """half-voxel ties of the 2x maps round to even, as the oracle does"""
    a_pred, a_file = _scaled(src, dst, angle)
    _check(pkg, _probs((c,) + src, seed=2), a_pred, a_file, dst, mode="nearest")


def _same_bits(a, b):
    """bit for bit, with every NaN counted as one value (the GPU returns its canonical NaN, not the payload it read)"""
    na, nb = a.isnan(), b.isnan()
    return torch.equal(na, nb) and torch.equal(a.masked_fill(na, 0.0).contiguous().view(torch.int32),
                                               b.masked_fill(nb, 0.0).contiguous().view(torch.int32))


def _specials(shape, seed=3):
    x = torch.randn(shape, generator=torch.Generator().manual_seed(seed))
    x[0, 1, 2, 3], x[0, 4, 5, 6], x[-1, 7, 8, 9], x[-1, 0, 0, 0] = -0.0, float("inf"), float("-inf"), float("nan")
    x[0, 3, 4:9, 2] = -0.0
    x[-1, -1, -1, -1] = float("nan")
    return x


@pytest.mark.parametrize("mode", ["trilinear", "nearest"])
def test_flips_permutations_shifts_and_identity_copy_exactly(pkg, mode):
    shape = (20, 24, 18)
    x = _specials((3,) + shape)
    xd = x.to(DEV)
    a0 = rc.file_affine((0.9375, 0.9375, 1.4), origin=(-12.5, 30.1, 4.0), lps=True)
    # orientation: the file's voxel v is the prediction's voxel (v[2], 19 - v[0], 23 - v[1])
    p, pshape = rc.flip_perm(shape, perm=(2, 0, 1), flips=(1, 2))
    pred = x.permute(0, 3, 1, 2).flip(2, 3).contiguous()
    got = pkg.prepost.resample_to_match(pred.to(DEV), a0 @ p, a0, shape, mode=mode)
    assert _same_bits(got.cpu(), x)
    # crop: the file is 6 voxels longer on each side of every axis; outside the box the prediction's edge extends (border)
    big = tuple(n + 12 for n in shape)
    got = pkg.prepost.resample_to_match(xd, a0 @ rc.crop((6, 6, 6)), a0, big, mode=mode)
    sel = [np.clip(np.arange(n) - 6, 0, m - 1) for n, m in zip(big, shape)]
    assert _same_bits(got.cpu(), x[:, sel[0]][:, :, sel[1]][:, :, :, sel[2]])
    # identical grids: copied without a kernel, and the kernel's own identity copy
    assert torch.equal(pkg.prepost.resample_to_match(xd, a0, a0, shape, mode=mode).view(torch.int32), xd.view(torch.int32))
    lib = pkg.lib.load_library()
    out = torch.empty_like(xd)
    eye = (pkg.lib.C.c_double * 12)(*np.eye(4)[:3].ravel().tolist())
    pkg.lib.check(lib.b200unet_resample_to_grid(xd.data_ptr(), 3, *shape, eye, pkg.prepost.resample_mode(mode), out.data_ptr(), *shape,
                                                pkg.lib.stream_ptr()), "resample_to_grid")
    assert _same_bits(out.cpu(), x)


def test_two_calls_are_bit_identical(pkg):
    a0, shape, a, pshape = rc.grid("sppin")
    x = _probs((2,) + pshape, seed=4).to(DEV)
    y1 = pkg.prepost.resample_to_match(x, a, a0, shape)
    y2 = pkg.prepost.resample_to_match(x, a, a0, shape)
    assert torch.equal(y1.view(torch.int32), y2.view(torch.int32))


def test_rejected_arguments(pkg):
    x = torch.zeros(129, 4, 4, 4, device=DEV)
    with pytest.raises(RuntimeError, match="1..128 channels"):
        pkg.prepost.resample_to_match(x, np.eye(4), np.eye(4), (5, 5, 5))
    bad = np.eye(4)
    bad[0, 0] = 0.0                                   # singular: no index map
    with pytest.raises(np.linalg.LinAlgError):
        pkg.prepost.resample_to_match(x[:2], bad, np.eye(4), (5, 5, 5))


# ------------------------------------------------------------------------------------------------ volumetric_predictions
class _Meta(torch.Tensor):
    pass


def _batch(pshape, grids, c_in=1, seed=5):
    """a [2, c_in, *pshape] MetaTensor-like batch on the device whose items come from the files (a_file, file_shape) and sit on the
    prediction grids a_pred, metadata batched as the collate function leaves it"""
    x = torch.randn((2, c_in) + pshape, generator=torch.Generator().manual_seed(seed)).to(DEV).as_subclass(_Meta)
    x.meta = {"filename_or_obj": ["a.nii.gz", "b.nii.gz"], "affine": torch.tensor(np.stack([g[2] for g in grids])),
              "original_affine": torch.tensor(np.stack([g[0] for g in grids])), "spatial_shape": torch.tensor([g[1] for g in grids])}
    return x


def _grids():
    """(file affine, file shape, prediction affine) of the two items: a resize with a crop offset, and a rotated, sheared grid"""
    out = []
    for shape, angle, shear, offset in (((30, 26, 20), 0.0, 0.0, (-2.0, 3.0, 1.0)), ((40, 36, 28), 0.2, 0.05, (1.0, -0.5, 0.25))):
        a_pred, a_file = _scaled((24, 24, 24), shape, angle, shear, offset)
        out.append((a_file, shape, a_pred))
    return out


def _check_predictions(pkg, res, plain, grids, interpolation):
    for i, (fn, p) in enumerate(res):
        a_file, shape, a_pred = grids[i]
        assert fn == ["a.nii.gz", "b.nii.gz"][i] and p.shape == (plain.shape[1],) + tuple(shape) and p.dtype == torch.float32
        ref = rc.oracle(plain[i].cpu().double().numpy(), pkg.prepost.index_map(a_pred, a_file), shape, interpolation)
        err = float(np.abs(p.cpu().double().numpy() - ref).max())
        assert err <= (0.0 if interpolation == "nearest" else 1e-6), (i, err)


@pytest.mark.parametrize("interpolation", ["trilinear", "nearest"])
def test_volumetric_predictions_resample_with_a_conv_model(pkg, interpolation):
    torch.manual_seed(0)
    model = nn.Conv3d(1, 3, kernel_size=3, padding=1).to(DEV)
    grids = _grids()
    x = _batch((24, 24, 24), grids)
    written = []
    res = pkg.predict.volumetric_predictions(model, [{"image": x}], "out", activation="sigmoid", resample=True,
                                             interpolation=interpolation, writer=lambda fn, t, d: written.append((fn, tuple(t.shape))))
    plain = pkg.predict.volumetric_predictions(model, [{"image": x}], "out", activation="sigmoid")
    with torch.no_grad():
        direct = torch.sigmoid(model(x.as_subclass(torch.Tensor)))
    assert all(torch.equal(p, direct[i]) for i, (_, p) in enumerate(plain))        # resample=False: as before
    _check_predictions(pkg, res, direct, grids, interpolation)
    assert written == [(fn, tuple(p.shape)) for fn, p in res]


def test_volumetric_predictions_resample_with_unet_behind_the_inferer(pkg):
    model = pkg.UNet3D(n_features=1, n_outputs=2, base_width=8).to(DEV)
    model.eval()
    inferer = pkg.SlidingWindowInferer(roi_size=(16, 16, 16), sw_batch_size=2, overlap=0.25)
    grids = _grids()
    x = _batch((24, 24, 24), grids)
    res = pkg.predict.volumetric_predictions(model, [{"image": x}], "out", activation="sigmoid", resample=True, inferer=inferer)
    plain = pkg.predict.volumetric_predictions(model, [{"image": x}], "out", activation="sigmoid", inferer=inferer)
    with torch.no_grad():
        direct = torch.sigmoid(inferer(x.as_subclass(torch.Tensor), model))
    assert all(p.shape == (2, 24, 24, 24) and torch.equal(p, direct[i]) for i, (_, p) in enumerate(plain))
    _check_predictions(pkg, res, direct, grids, "trilinear")
