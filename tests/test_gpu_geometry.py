"""Device crop + resize (``augment.CropForegroundd`` / ``Resized``, ``csrc/foreground.cu`` and the per-sample sources of
``csrc/augment.cu``) against numpy and the fp64 oracle (tests/geometry_oracle.py): the percentile threshold bit for bit, the
foreground boxes exactly, the one composed resample, bit identities, and training on a loader of different-size items."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import geometry_oracle  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
KEYS = ("image", "label")
PERCENTILES = (0.0, 0.1, 0.5, 0.9, 0.999, 1.0)


def _same_value(a: np.ndarray, b: np.ndarray) -> bool:
    """bit for bit, with -0 counted as +0 (numpy's partition leaves either) and every NaN as one value"""
    na, nb = np.isnan(a), np.isnan(b)
    a0, b0 = np.where(na, 0, a + np.float32(0)), np.where(nb, 0, b + np.float32(0))
    return bool((na == nb).all() and (a0.astype(np.float32).view(np.int32) == b0.astype(np.float32).view(np.int32)).all())


def _mri_like(shape, seed):
    """4 channels: mostly exact zeros with a N(0, 1) core, heavy ties (integers 0..5), a constant, and N(0, 1) with a NaN"""
    g = torch.Generator().manual_seed(seed)
    d, h, w = shape
    x = torch.zeros((4,) + shape)
    core = torch.randn(shape, generator=g)
    keep = torch.rand(shape, generator=g) < 0.25
    x[0] = torch.where(keep, core, torch.zeros(()))
    x[1] = torch.randint(0, 6, shape, generator=g).float()
    x[2] = 3.5
    x[3] = torch.randn(shape, generator=g)
    x[3].view(-1)[(d * h * w) // 2] = float("nan")
    return x


def test_threshold_matches_numpy_bit_for_bit(pkg):
    aug = pkg.augment
    shapes = [(1, 1, 1), (1, 1, 2), (1, 1, 7), (10, 10, 10), (240, 240, 155)]
    xs = [_mri_like(s, i) for i, s in enumerate(shapes)]
    xd = [x.to(DEV) for x in xs]
    for p in PERCENTILES:
        comp = aug.Compose([aug.CropForegroundd("image", foreground_percentile=p), aug.Resized("image", spatial_size=(4, 4, 4))])
        comp({"image": xd})
        got = comp.last_params["threshold"].cpu().numpy()
        ref = np.array([geometry_oracle.threshold(x.numpy(), p) for x in xs], dtype=np.float32)
        assert _same_value(got, ref), (p, got, ref)
        assert np.isnan(got[:, 3]).all() and (got[:, 2] == 3.5).all()


def _box_cases():
    """(C, D, H, W) fp32 volumes of background -1 with foreground (> 0): touching each face, one voxel, none"""
    shape = (2, 9, 12, 7)
    out = []
    for face in range(6):
        x = torch.full(shape, -1.0)
        ax, hi = face // 2, face % 2
        idx = [slice(3, 5), slice(4, 8), slice(2, 4)]
        idx[ax] = slice(shape[1 + ax] - 2, shape[1 + ax]) if hi else slice(0, 2)
        x[(face % 2,) + tuple(idx)] = 2.0
        out.append(x)
    one = torch.full(shape, -1.0)
    one[1, 4, 5, 3] = 0.5
    out += [one, torch.full(shape, -1.0), torch.rand((2, 5, 13, 11), generator=torch.Generator().manual_seed(4)) - 0.5]
    return out


@pytest.mark.parametrize("allow_smaller", [True, False])
@pytest.mark.parametrize("percentile", [None, 0.9])
def test_boxes_match_numpy(pkg, allow_smaller, percentile):
    aug = pkg.augment
    xs = _box_cases()
    comp = aug.Compose([aug.CropForegroundd("image", foreground_percentile=percentile, margin=1, allow_smaller=allow_smaller),
                        aug.Resized("image", spatial_size=(6, 6, 6))])
    comp({"image": [x.to(DEV) for x in xs]})
    box, empty = comp.last_params["box"].cpu().numpy(), comp.last_params["empty"].cpu().numpy()
    for i, x in enumerate(xs):
        ref, ref_empty = geometry_oracle.foreground_box(x.numpy(), percentile, 1, allow_smaller)
        assert box[i].tolist() == ref.tolist() and bool(empty[i]) == ref_empty, (i, box[i], ref)
    if percentile is None:
        assert empty.tolist() == [0] * 7 + [1, 0]
        if not allow_smaller:
            assert (box[:6, :, 0] < 0).any() and (box[:6, :, 1] > np.array([9, 12, 7])).any()


def _brats_like(shape, n_labels, seed):
    """N(0, 1) foreground in an off-centre sub-box, background -5 around it, and a random uint8 one-hot-like label"""
    g = torch.Generator().manual_seed(seed)
    x = torch.full((4,) + shape, -5.0)
    lo = [s // 5 for s in shape]
    hi = [s - s // 4 for s in shape]
    x[:, lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = torch.randn((4,) + tuple(b - a for a, b in zip(lo, hi)), generator=g)
    lab = (torch.rand((n_labels,) + shape, generator=g) > 0.6).to(torch.uint8)
    return x, lab


def _label_ties(src, size, band=1e-4):
    """output voxels whose fp64 source coordinate lies within ``band`` voxels of a rounding tie (border padding)"""
    src = torch.minimum(src.clamp(min=0), torch.tensor(size, dtype=torch.float64) - 1)
    return ((src - src.floor() - 0.5).abs() < band).any(-1)


@pytest.mark.parametrize("out_size", [(24, 28, 20), (40, 36, 44)])
def test_resample_matches_fp64_oracle(pkg, out_size):
    aug = pkg.augment
    shapes = [(37, 41, 30), (45, 33, 39)]
    data = [_brats_like(s, 3, i) for i, s in enumerate(shapes)]
    comp = aug.Compose([aug.CropForegroundd(KEYS, foreground_percentile=0.1), aug.Resized(KEYS, spatial_size=out_size),
                        aug.RandFlipd(KEYS, prob=0.5, spatial_axis=0),
                        aug.RandRotated(KEYS, range_x=0.2, range_y=0.2, range_z=0.2, prob=1.0),
                        aug.NormalizeIntensityd("image", channel_wise=True),
                        aug.RandScaleIntensityd("image", factors=0.1, prob=1.0),
                        aug.RandShiftIntensityd("image", offsets=0.1, prob=1.0)]).set_random_state(3)
    out = comp({"image": [x.to(DEV) for x, _ in data], "label": [lab.to(DEV) for _, lab in data]})
    p = comp.last_params
    assert out["image"].shape == (2, 4) + out_size and out["label"].shape == (2, 3) + out_size
    box = p["box"].cpu().numpy()
    for i, (x, _) in enumerate(data):
        ref_box, _ = geometry_oracle.foreground_box(x.numpy(), 0.1, 1, True)
        assert box[i].tolist() == ref_box.tolist()
        assert all(b - a < s for (a, b), s in zip(box[i], shapes[i]))           # a real crop
    ref, ref_l = geometry_oracle.geometry([x for x, _ in data], [lab for _, lab in data], p)
    got = out["image"].cpu().double()
    err = (got - ref).abs().max().item()
    print("geometry resample %s: max abs %.3e" % (out_size, err))
    assert err <= 1.5e-4
    for i in range(2):
        src = geometry_oracle.source_coordinates(p["affine"][i], box[i], out_size)
        tie = _label_ties(src, shapes[i])[None].expand_as(ref_l[i])
        mism = out["label"][i].cpu().double() != ref_l[i]
        assert not (mism & ~tie).any() and tie.double().mean().item() < 1e-3


def _same_bits(a, b):
    na, nb = a.isnan(), b.isnan()
    return torch.equal(na, nb) and torch.equal(a.masked_fill(na, 0.0).contiguous().view(torch.int32),
                                               b.masked_fill(nb, 0.0).contiguous().view(torch.int32))


def test_bit_identities(pkg):
    aug = pkg.augment
    x, lab = _brats_like((20, 24, 18), 2, 7)
    x[0, 10, 12, 9] = -0.0
    xd, ld = x.to(DEV), lab.to(DEV)
    # whole-volume box (foreground reaches every face), spatial_size = the input's, nothing drawn: the input itself
    full = torch.randn((4, 20, 24, 18), generator=torch.Generator().manual_seed(1)).to(DEV)
    for crop in ([], [aug.CropForegroundd(KEYS, foreground_percentile=0.0)]):
        comp = aug.Compose(crop + [aug.Resized(KEYS, spatial_size=(20, 24, 18)), aug.RandFlipd(KEYS, prob=0.0),
                                   aug.RandRotated(KEYS, range_x=0.3, prob=0.0)])
        out = comp({"image": full[None], "label": ld[None]})
        assert comp.last_params["box"][0].tolist() == [[0, 20], [0, 24], [0, 18]]
        assert _same_bits(out["image"][0], full) and torch.equal(out["label"][0], ld)
    # a list of two different sizes = each sample alone (the draws are fixed: prob 1, one-point ranges)
    y, laby = _brats_like((26, 19, 23), 2, 8)
    comp = aug.Compose([aug.CropForegroundd(KEYS, foreground_percentile=0.1), aug.Resized(KEYS, spatial_size=(16, 20, 12)),
                        aug.RandFlipd(KEYS, prob=1.0, spatial_axis=1), aug.RandRotated(KEYS, range_x=(0.1, 0.1), prob=1.0),
                        aug.NormalizeIntensityd("image", channel_wise=True)])
    both = comp({"image": [xd, y.to(DEV)], "label": [ld, laby.to(DEV)]})
    alone = [comp({"image": [a], "label": [b]}) for a, b in ((xd, ld), (y.to(DEV), laby.to(DEV)))]
    for i in range(2):
        assert _same_bits(both["image"][i], alone[i]["image"][0]) and torch.equal(both["label"][i], alone[i]["label"][0])
    # one 5-D batch = the same samples as a list
    z = torch.stack([xd, xd + 1])
    zl = torch.stack([ld, ld])
    a = comp({"image": z, "label": zl})
    b = comp({"image": list(z), "label": list(zl)})
    assert _same_bits(a["image"], b["image"]) and torch.equal(a["label"], b["label"])
    # the same seed twice, with random draws
    comp = aug.Compose([aug.CropForegroundd(KEYS, foreground_percentile=0.1), aug.Resized(KEYS, spatial_size=(16, 20, 12)),
                        aug.RandFlipd(KEYS, prob=0.5), aug.RandRotated(KEYS, range_x=0.2, range_z=0.2, prob=0.5),
                        aug.NormalizeIntensityd("image"), aug.RandShiftIntensityd("image", offsets=0.1, prob=1.0)])
    r = [comp.set_random_state(5)({"image": [xd, y.to(DEV)], "label": [ld, laby.to(DEV)]}) for _ in range(2)]
    assert _same_bits(r[0]["image"], r[1]["image"]) and torch.equal(r[0]["label"], r[1]["label"])


KW = dict(n_features=4, n_outputs=3, base_width=8, encoder_blocks=[1, 1, 1], decoder_blocks=[1, 1, 1], dropout=0.0)
SECTION = {"name": "SegmentationDataset", "desired_shape": [32, 32, 32], "labels": [2, 1, 4], "resample": True,
           "crop_foreground": True, "normalization": "NormalizeIntensityD", "normalization_kwargs": {"channel_wise": True},
           "training": {"spatial_augmentations": [{"name": "RandFlipD", "spatial_axis": 0, "prob": 0.5},
                                                  {"name": "RandRotateD", "prob": 0.5, "range_x": 0.2}]}}


@pytest.mark.parametrize("graph", [False, True])
def test_epoch_training_on_different_size_items(pkg, graph):
    aug = pkg.augment
    items = []
    for i, s in enumerate([(30, 34, 28), (36, 30, 32), (28, 40, 35), (33, 33, 30)]):
        x, lab = _brats_like(s, 3, 20 + i)
        items.append({"image": x, "label": lab})
    loader = torch.utils.data.DataLoader(items, batch_size=2, collate_fn=aug.list_collate, pin_memory=True)
    comp, rest = aug.build_device_transform(SECTION, geometry=True)
    assert rest["training"]["crop_foreground"] is False and rest["training"]["desired_shape"] is None
    torch.manual_seed(0)
    model = pkg.UNet3D(precision="bf16", deterministic=True, **KW).to(DEV)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    avg = pkg.train.epoch_training(loader, model, pkg.DiceLoss(sigmoid=True), opt, epoch=0, n_gpus=1, print_frequency=0,
                                   use_cuda_graph=graph, device_transform=comp.set_random_state(0))
    torch.cuda.synchronize()
    assert np.isfinite(avg) and 0.0 < avg < 1.0
    assert all(torch.isfinite(p).all() for p in model.parameters())
    assert comp.last_params["box"].shape == (2, 3, 2)
