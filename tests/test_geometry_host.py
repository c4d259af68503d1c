"""Host side of the device crop + resize (``augment.CropForegroundd`` / ``Resized``): the fp64 oracle of the composed map
(tests/geometry_oracle.py) against ``F.interpolate``, numpy's percentile index arithmetic, the BraTS and SPPIN dataset
sections rewritten by ``build_device_transform(geometry=True)``, ``list_collate`` and the options that raise."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import geometry_oracle  # noqa: E402

KEYS = ("image", "label")

# the "dataset" sections of the reference's examples/brats2020/brats2020_config.json and examples/sppin/sppin_config.json,
# restated (the SPPIN one with its augmentations)
BRATS_DATASET = {
    "name": "SegmentationDataset", "desired_shape": [128, 128, 128], "labels": [2, 1, 4], "setup_label_hierarchy": True,
    "normalization": "NormalizeIntensityD", "normalization_kwargs": {"channel_wise": True, "nonzero": False},
    "resample": True, "crop_foreground": True,
}
SPPIN_DATASET = {
    "name": "SegmentationDatasetPersistent", "desired_shape": [192, 192, 192], "labels": [1], "orientation": "RAS",
    "normalization": "NormalizeIntensityD", "normalization_kwargs": {"channel_wise": True, "nonzero": False},
    "resample": True, "crop_foreground": True, "foreground_percentile": 0.9,
    "training": {
        "spatial_augmentations": [{"name": "RandFlipD", "spatial_axis": 0, "prob": 0.5},
                                  {"name": "RandFlipD", "spatial_axis": 1, "prob": 0.5},
                                  {"name": "RandRotateD", "prob": 0.5, "range_x": 0.2, "range_y": 0.2, "range_z": 0.2}],
        "intensity_augmentations": [{"name": "RandScaleIntensityD", "factors": 0.1, "prob": 1.0},
                                    {"name": "RandShiftIntensityD", "offsets": 0.1, "prob": 1.0}],
    },
}
GEOMETRY_KEYS = ("crop_foreground", "foreground_percentile", "desired_shape", "resample", "random_crop")


@pytest.fixture(scope="module")
def aug(pkg):
    return pkg.augment


@pytest.mark.parametrize("size,out", [((11, 17, 9), (8, 20, 13)), ((16, 16, 16), (16, 16, 16)), ((5, 40, 7), (12, 10, 7))])
def test_oracle_whole_box_without_augmentation_is_interpolate(size, out):
    x = torch.randn((3,) + size, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    box = [[0, s] for s in size]
    src = geometry_oracle.source_coordinates(torch.eye(4, dtype=torch.float64)[:3], box, out)
    got = geometry_oracle.sample(x, src, "border", "bilinear")
    ref = F.interpolate(x[None], size=out, mode="trilinear", align_corners=False)[0]
    assert (got - ref).abs().max().item() < 1e-12


def _lerp32(a, b, t):
    """numpy's _lerp on fp32 scalars: a + (b - a) t, or b - (b - a)(1 - t) where t >= 0.5"""
    diff = np.float32(b) - np.float32(a)
    return np.float32(b) - diff * (np.float32(1) - t) if t >= 0.5 else np.float32(a) + diff * t


@pytest.mark.parametrize("size", [1, 2, 3, 7, 10, 1000, 4097, 240 * 240 * 155])
def test_percentile_index_reproduces_numpy(aug, size):
    g = np.random.default_rng(size)
    x = g.standard_normal(size).astype(np.float32)
    x[g.random(size) < 0.5] = 0.0                      # heavy ties
    xs = np.sort(x)
    for p in (0.0, 0.1, 0.5, 0.9, 0.999, 1.0, 0.25, 1.0 / 3.0):
        lo, hi, gamma = aug.percentile_index(size, p)
        assert 0 <= lo <= hi <= size - 1 and hi - lo <= 1 and isinstance(gamma, np.float32)
        got = _lerp32(xs[lo], xs[hi], gamma)
        ref = np.percentile(x, p * 100)
        assert ref.dtype == np.float32 and got.view(np.int32) == ref.view(np.int32), (size, p, got, ref)


def test_foreground_box_restatement():
    x = np.full((2, 6, 7, 8), -1.0, dtype=np.float32)
    x[1, 2, 3, 4] = 5.0                                            # a single voxel
    box, empty = geometry_oracle.foreground_box(x, None, 1, True)
    assert not empty and box.tolist() == [[1, 4], [2, 5], [3, 6]]
    x[0, 0, 6, 7] = 2.0                                            # touching three faces: clipped, or past the edge
    assert geometry_oracle.foreground_box(x, None, 1, True)[0].tolist() == [[0, 4], [2, 7], [3, 8]]
    assert geometry_oracle.foreground_box(x, None, 1, False)[0].tolist() == [[-1, 4], [2, 8], [3, 9]]
    box, empty = geometry_oracle.foreground_box(np.zeros((1, 3, 4, 5), np.float32), None, 1, True)
    assert empty and box.tolist() == [[0, 3], [0, 4], [0, 5]]


def _split_kwargs(section, split):
    """the dataset kwargs of one split as the reference's build_data_loaders assembles them (unet3d/scripts/script_utils.py:
    107-121,140-142; inference reads the validation entries, :155-176): the split's entries plus the top level's.  A key in
    both is a duplicate keyword argument there (TypeError)."""
    top = {k: v for k, v in section.items() if k not in ("name", "training", "validation")}
    extra = section.get(split) or {}
    assert not set(extra) & set(top), "duplicate keyword arguments: %s" % sorted(set(extra) & set(top))
    return {**extra, **top}


@pytest.mark.parametrize("section,percentile", [(BRATS_DATASET, 0.1), (SPPIN_DATASET, 0.9),
                                                (dict(SPPIN_DATASET, validation={"random_crop": False}), 0.9)])
def test_geometry_rewrite_keeps_validation_and_inference(aug, section, percentile):
    compose, rest = aug.build_device_transform(section, geometry=True)
    assert _split_kwargs(rest, "validation") == _split_kwargs(section, "validation")
    train = _split_kwargs(rest, "training")
    assert train["crop_foreground"] is False and train["desired_shape"] is None and train["normalization"] is None
    assert not {"foreground_percentile", "resample", "spatial_augmentations", "intensity_augmentations"} & set(train)
    names = [type(t).__name__ for t in compose.transforms]
    assert names[:2] == ["CropForegroundd", "Resized"]
    assert compose.crop.percentile == percentile and compose.crop.margin == 1 and compose.crop.allow_smaller
    assert compose.resize.spatial_size == tuple(section["desired_shape"]) and compose.spatial_keys == KEYS
    # without geometry: what build_device_transform returned before the option existed
    plain, rest0 = aug.build_device_transform(section)
    assert rest0 == aug.build_device_transform(section, geometry=False)[1]
    assert [type(t).__name__ for t in plain.transforms] == names[2:] and plain.resize is None
    assert all(rest0.get(k) == section.get(k) for k in GEOMETRY_KEYS)


def test_geometry_options_that_raise(aug):
    with pytest.raises(NotImplementedError, match="random_crop"):
        aug.build_device_transform(dict(BRATS_DATASET, random_crop=True), geometry=True)
    with pytest.raises(NotImplementedError, match="ResizeWithPadOrCropD"):
        aug.build_device_transform(dict(BRATS_DATASET, resample=False), geometry=True)
    aug.build_device_transform(dict(BRATS_DATASET, random_crop=True))          # the default leaves both to the host
    aug.build_device_transform(dict(BRATS_DATASET, resample=False))
    with pytest.raises(NotImplementedError, match="select_fn"):
        aug.CropForegroundd(KEYS, select_fn=lambda x: x > 0)
    with pytest.raises(NotImplementedError, match="source_key"):
        aug.CropForegroundd(KEYS, source_key="label")
    with pytest.raises(NotImplementedError, match="label"):
        aug.Resized(KEYS, spatial_size=(8, 8, 8), mode=("trilinear", "trilinear"))
    with pytest.raises(NotImplementedError, match="image"):
        aug.Resized(KEYS, spatial_size=(8, 8, 8), mode=("area", "nearest"))
    with pytest.raises(NotImplementedError, match="spatial_size"):
        aug.Resized(KEYS, spatial_size=(8, -1, 8))
    crop, resize = aug.CropForegroundD(KEYS, foreground_percentile=0.1), aug.ResizeD(KEYS, spatial_size=(8, 8, 8))
    flip = aug.RandFlipd(KEYS, prob=0.5)
    aug.Compose([crop, resize, flip, aug.NormalizeIntensityd("image")])
    aug.Compose([resize, flip])
    for bad in ([resize, crop], [crop, resize, resize], [crop, crop, resize], [flip, crop, resize], [flip, resize], [crop],
                [crop, flip]):
        with pytest.raises(ValueError, match="order|Resized"):
            aug.Compose(bad)
    with pytest.raises(ValueError, match="keys"):
        aug.Compose([aug.CropForegroundd("image"), resize, flip])
    assert aug.CropForegroundD is aug.CropForegroundd and aug.ResizeD is aug.Resized


def test_list_collate_keeps_samples_apart(aug):
    items = [{"image": torch.zeros(4, 5, 6, 7), "label": torch.zeros(3, 5, 6, 7, dtype=torch.uint8), "id": 0},
             {"image": torch.ones(4, 8, 6, 5), "label": torch.ones(3, 8, 6, 5, dtype=torch.uint8), "id": 1}]
    batch = aug.list_collate(items)
    assert [tuple(t.shape) for t in batch["image"]] == [(4, 5, 6, 7), (4, 8, 6, 5)]
    assert [tuple(t.shape) for t in batch["label"]] == [(3, 5, 6, 7), (3, 8, 6, 5)]
    assert torch.equal(batch["id"], torch.tensor([0, 1]))
    loader = torch.utils.data.DataLoader(items, batch_size=2, collate_fn=aug.list_collate)
    assert [tuple(t.shape) for t in next(iter(loader))["image"]] == [(4, 5, 6, 7), (4, 8, 6, 5)]
