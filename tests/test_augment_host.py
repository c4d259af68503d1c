"""Host side of the device augmentation (``augment.py``): parameter sampling, the composed affine, reading a config's
``dataset`` section, the options that raise, and the fp64 oracle (tests/augment_oracle.py) against an explicit loop."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import augment_oracle  # noqa: E402

SPATIAL = (24, 40, 33)

# examples/sppin/sppin_config.json "dataset" section of the reference, restated
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


@pytest.fixture(scope="module")
def aug(pkg):
    return pkg.augment


def _all(aug, prob, **kw):
    keys = ("image", "label")
    return aug.Compose([aug.RandFlipd(keys, prob=prob, spatial_axis=0), aug.RandRotated(keys, range_x=0.2, range_y=0.3, range_z=0.4,
                                                                                        prob=prob, **kw),
                        aug.NormalizeIntensityd(("image",)), aug.RandScaleIntensityd(("image",), factors=0.1, prob=prob),
                        aug.RandShiftIntensityd(("image",), offsets=0.1, prob=prob)]).set_random_state(0)


def test_prob_zero_draws_nothing_and_prob_one_everything(aug):
    p = _all(aug, 0.0).draw(4, 3, SPATIAL)
    assert all(not r["do"] for s in p["transforms"] for r in s if r["name"] != "NormalizeIntensityd")
    assert torch.equal(p["affine"], torch.eye(4, dtype=torch.float64)[:3].expand(4, 3, 4))
    assert torch.equal(p["coef"][..., 0], torch.ones(4, 3, dtype=torch.float64)) and not p["coef"][..., 1].any()
    q = _all(aug, 1.0).draw(4, 3, SPATIAL)
    assert all(r["do"] for s in q["transforms"] for r in s)
    for s in q["transforms"]:
        rot = s[1]["angles"]
        assert all(0 < abs(a) <= lim for a, lim in zip(rot, (0.2, 0.3, 0.4)))
        assert all(abs(v) <= 0.1 for v in s[3]["factors"] + s[4]["offsets"])


def test_scalar_and_pair_ranges(aug):
    g = aug.Compose([aug.RandRotated("image", range_x=(0.1, 0.3), range_y=0.05, range_z=(-0.4, -0.39), prob=1.0),
                     aug.RandScaleIntensityd("image", factors=(0.5, 0.6), prob=1.0),
                     aug.RandShiftIntensityd("image", offsets=2.0, prob=1.0)]).set_random_state(3)
    p = g.draw(64, 2, SPATIAL)
    ang = np.array([s[0]["angles"] for s in p["transforms"]])
    assert (ang[:, 0] >= 0.1).all() and (ang[:, 0] <= 0.3).all()
    assert (np.abs(ang[:, 1]) <= 0.05).all() and (ang[:, 1] < 0).any() and (ang[:, 1] > 0).any()
    assert (ang[:, 2] >= -0.4).all() and (ang[:, 2] <= -0.39).all()
    f = np.array([s[1]["factors"] for s in p["transforms"]])
    o = np.array([s[2]["offsets"] for s in p["transforms"]])
    assert (f >= 0.5).all() and (f <= 0.6).all() and (np.abs(o) <= 2.0).all() and (o < 0).any() and (o > 0).any()
    assert (f[:, 0] == f[:, 1]).all()                                   # not channel_wise: one draw for all channels
    # the composed coefficients: x * (1 + f) + o
    assert np.allclose(p["coef"][..., 0].numpy(), 1 + f) and np.allclose(p["coef"][..., 1].numpy(), o)
    cw = aug.Compose([aug.RandScaleIntensityd("image", factors=0.1, prob=1.0, channel_wise=True)]).set_random_state(3)
    fc = np.array([s[0]["factors"] for s in cw.draw(8, 4, SPATIAL)["transforms"]])
    assert fc.shape == (8, 4) and len(np.unique(fc)) == 32


def test_draws_are_per_sample_and_reproducible(aug):
    a = _all(aug, 0.5).draw(16, 4, SPATIAL)
    b = _all(aug, 0.5).draw(16, 4, SPATIAL)
    assert a["transforms"] == b["transforms"] and torch.equal(a["affine"], b["affine"]) and torch.equal(a["coef"], b["coef"])
    fired = [[r["do"] for r in s] for s in a["transforms"]]
    assert len({tuple(f) for f in fired}) > 1                          # samples draw independently
    angles = [s[1]["angles"] for s in a["transforms"] if s[1]["do"]]
    assert len(set(angles)) == len(angles) > 1
    c = _all(aug, 0.5).set_random_state(1).draw(16, 4, SPATIAL)
    assert c["transforms"] != a["transforms"]
    # the generator advances: a second batch differs from the first
    g = _all(aug, 0.5)
    assert g.draw(16, 4, SPATIAL)["transforms"] != g.draw(16, 4, SPATIAL)["transforms"]


def _create_rotate(x, y, z):
    """MONAI create_rotate(3, (x, y, z)) restated as 4 x 4 homogeneous matrices."""
    rx = np.array([[1, 0, 0, 0], [0, math.cos(x), -math.sin(x), 0], [0, math.sin(x), math.cos(x), 0], [0, 0, 0, 1]])
    ry = np.array([[math.cos(y), 0, math.sin(y), 0], [0, 1, 0, 0], [-math.sin(y), 0, math.cos(y), 0], [0, 0, 0, 1]])
    rz = np.array([[math.cos(z), -math.sin(z), 0, 0], [math.sin(z), math.cos(z), 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    return rx @ ry @ rz


def test_single_rotation_matches_create_rotate(aug):
    angles = (0.11, -0.17, 0.05)
    g = aug.Compose([aug.RandRotated("image", range_x=(angles[0],) * 2, range_y=(angles[1],) * 2, range_z=(angles[2],) * 2,
                                     prob=1.0)])
    p = g.draw(1, 1, SPATIAL)
    assert np.allclose(p["transforms"][0][0]["angles"], angles, atol=1e-15)
    c = (np.array(SPATIAL, dtype=np.float64) - 1) / 2
    to_c, from_c = np.eye(4), np.eye(4)
    to_c[:3, 3], from_c[:3, 3] = -c, c
    ref = from_c @ _create_rotate(*angles) @ to_c                       # source = c + R (p - c)
    assert np.allclose(p["affine"][0].numpy(), ref[:3], atol=1e-12)
    assert np.allclose(p["matrices"][0][0].numpy(), ref, atol=1e-12)


def test_composed_affine_is_the_product_in_application_order(aug):
    keys = ("image", "label")
    g = aug.Compose([aug.RandFlipd(keys, prob=1.0, spatial_axis=0), aug.RandRotated(keys, range_x=0.2, range_z=0.3, prob=1.0),
                     aug.RandFlipd(keys, prob=1.0, spatial_axis=(1, 2))]).set_random_state(5)
    p = g.draw(3, 1, SPATIAL)
    for i in range(3):
        m = p["matrices"][i].numpy()
        assert m.shape == (3, 4, 4)
        assert np.allclose(p["affine"][i].numpy(), (m[0] @ m[1] @ m[2])[:3], atol=1e-12)
    # semantics: the first flip alone maps output index p to source (D - 1 - p_d, p_h, p_w)
    f = aug.Compose([aug.RandFlipd(keys, prob=1.0, spatial_axis=0)]).draw(1, 1, SPATIAL)["affine"][0].numpy()
    assert np.array_equal(f @ np.array([2.0, 5.0, 7.0, 1.0]), [SPATIAL[0] - 3, 5, 7])
    # flip(0) then flip(0) is the identity; spatial_axis=None flips all three axes
    ff = aug.Compose([aug.RandFlipd(keys, prob=1.0, spatial_axis=0)] * 2).draw(1, 1, SPATIAL)["affine"][0]
    assert torch.equal(ff, torch.eye(4, dtype=torch.float64)[:3])
    fa = aug.Compose([aug.RandFlipd(keys, prob=1.0)]).draw(1, 1, SPATIAL)["affine"][0].numpy()
    assert np.array_equal(np.diag(fa[:, :3]), [-1, -1, -1]) and np.array_equal(fa[:, 3], np.array(SPATIAL) - 1)


def test_build_device_transform_reads_the_sppin_dataset_section(aug):
    compose, rest = aug.build_device_transform(SPPIN_DATASET)
    t = compose.transforms
    assert [type(x).__name__ for x in t] == ["RandFlipd", "RandFlipd", "RandRotated", "NormalizeIntensityd", "RandScaleIntensityd",
                                             "RandShiftIntensityd"]
    assert t[0].axes == (0,) and t[1].axes == (1,) and t[0].prob == t[1].prob == t[2].prob == 0.5
    assert t[2].ranges == ((-0.2, 0.2),) * 3 and compose.padding_mode == "border"
    assert t[3].channel_wise and not t[3].nonzero
    assert t[4].range == (-0.1, 0.1) and t[5].range == (-0.1, 0.1) and t[4].prob == t[5].prob == 1.0
    assert compose.spatial_keys == ("image", "label")
    assert "normalization" not in rest and "normalization_kwargs" not in rest
    assert rest["training"] == {"normalization": None}
    assert rest["validation"] == {"normalization": "NormalizeIntensityD", "normalization_kwargs": {"channel_wise": True, "nonzero": False}}
    assert {k: v for k, v in rest.items() if k not in ("training", "validation")} == \
        {k: v for k, v in SPPIN_DATASET.items() if k not in ("normalization", "normalization_kwargs", "training")}
    assert SPPIN_DATASET["training"]["spatial_augmentations"]                # the input is not modified
    # the reference's default normalisation is "zero_mean"; no augmentations gives a Compose of the z-score alone
    only, _ = aug.build_device_transform({"name": "SegmentationDataset"})
    assert [type(x).__name__ for x in only.transforms] == ["NormalizeIntensityd"]
    assert aug.RandFlipD is aug.RandFlipd and aug.RandRotateD is aug.RandRotated and aug.NormalizeIntensityD is aug.NormalizeIntensityd
    assert aug.RandScaleIntensityD is aug.RandScaleIntensityd and aug.RandShiftIntensityD is aug.RandShiftIntensityd


def _split_kwargs(section, split):
    """the dataset kwargs of one split as the reference assembles them (unet3d/scripts/script_utils.py:107-121,140-142 for
    training and validation; :155-176 for inference, which reads the validation entries): the split's entries plus the top
    level's.  A key in both is a duplicate keyword argument there (TypeError)."""
    top = {k: v for k, v in section.items() if k not in ("name", "training", "validation")}
    extra = section.get(split) or {}
    assert not set(extra) & set(top), "duplicate keyword arguments: %s" % sorted(set(extra) & set(top))
    return {**extra, **top}


def _host_normalization(kwargs):
    """(normalization, normalization_kwargs) the reference's dataset applies (segmentation.py:77-87 defaults)"""
    return kwargs.get("normalization", "zero_mean"), kwargs.get("normalization_kwargs") or {}


@pytest.mark.parametrize("section", [
    SPPIN_DATASET,
    dict(SPPIN_DATASET, validation={"random_crop": False}),
    {"name": "SegmentationDataset", "desired_shape": [64, 64, 64], "training": {"spatial_augmentations": [
        {"name": "RandFlipD", "spatial_axis": 2, "prob": 0.5}]}},                                  # default z-score
    {"normalization": None, "training": {"intensity_augmentations": [{"name": "RandShiftIntensityD", "offsets": 0.1}]}},
])
def test_rewritten_dataset_section_keeps_validation_and_inference_normalised(aug, section):
    """Only the training dataset hands its z-score to the device: validation and inference datasets built from the rewritten
    section normalise exactly as those built from the original one."""
    compose, rest = aug.build_device_transform(section)
    val, original = _split_kwargs(rest, "validation"), _split_kwargs(section, "validation")   # inference reads these too
    assert _host_normalization(val) == _host_normalization(original)
    other = ("normalization", "normalization_kwargs")
    assert {k: v for k, v in val.items() if k not in other} == {k: v for k, v in original.items() if k not in other}
    train = _split_kwargs(rest, "training")
    assert train["normalization"] is None
    assert "spatial_augmentations" not in train and "intensity_augmentations" not in train
    # the device applies what the host training dataset no longer does
    norm, kw = _host_normalization(_split_kwargs(section, "training"))
    dev = [t for t in compose.transforms if t.kind == "normalize"]
    if norm is None:
        assert not dev
    else:
        assert len(dev) == 1 and dev[0].channel_wise == bool(kw.get("channel_wise")) and dev[0].nonzero == bool(kw.get("nonzero"))


def test_unsupported_options_raise(aug):
    keys = ("image", "label")
    with pytest.raises(NotImplementedError, match="keep_size"):
        aug.RandRotated(keys, range_x=0.1, keep_size=False)
    with pytest.raises(NotImplementedError, match="align_corners"):
        aug.RandRotated(keys, range_x=0.1, align_corners=True)
    with pytest.raises(NotImplementedError, match="padding_mode"):
        aug.RandRotated(keys, range_x=0.1, padding_mode="reflection")
    with pytest.raises(NotImplementedError, match="label"):
        aug.RandRotated(keys, range_x=0.1, mode="bilinear")              # would apply bilinear to the label too
    with pytest.raises(NotImplementedError, match="label"):
        aug.RandRotated(keys, range_x=0.1, mode=("bilinear", "bilinear"))
    aug.RandRotated(keys, range_x=0.1, mode=("bilinear", "nearest"))
    with pytest.raises(NotImplementedError, match="image"):
        aug.RandRotated(keys, range_x=0.1, mode=("nearest", "nearest"))
    with pytest.raises(NotImplementedError, match="subtrahend"):
        aug.NormalizeIntensityd("image", subtrahend=1.0)
    with pytest.raises(NotImplementedError, match="RandAffineD"):
        aug.build_device_transform({"training": {"spatial_augmentations": [{"name": "RandAffineD", "prob": 0.1}]}})
    with pytest.raises(NotImplementedError, match="ScaleIntensityRange"):
        aug.build_device_transform({"normalization": "ScaleIntensityRange"})
    with pytest.raises(ValueError, match="order"):
        aug.Compose([aug.NormalizeIntensityd("image"), aug.RandFlipd(keys, prob=1.0)])
    with pytest.raises(ValueError, match="order"):
        aug.Compose([aug.RandShiftIntensityd("image", offsets=0.1), aug.NormalizeIntensityd("image")])
    with pytest.raises(ValueError, match="keys"):
        aug.Compose([aug.RandShiftIntensityd(keys, offsets=0.1)])
    with pytest.raises(ValueError, match="keys"):
        aug.Compose([aug.RandFlipd(keys, prob=1.0), aug.RandFlipd("image", prob=1.0)])
    with pytest.raises(ValueError, match="padding_mode"):
        aug.Compose([aug.RandRotated(keys, range_x=0.1), aug.RandRotated(keys, range_x=0.1, padding_mode="zeros")])
    with pytest.raises(ValueError, match="spatial_axis"):
        aug.RandFlipd(keys, spatial_axis=3)
    with pytest.raises(RuntimeError, match="CUDA"):
        aug.Compose([aug.RandFlipd(keys, prob=1.0)])({"image": torch.zeros(1, 1, 4, 4, 4), "label": torch.zeros(1, 1, 4, 4, 4)})


def test_epoch_training_rejects_a_device_transform_without_a_device(pkg, aug):
    model = torch.nn.Conv3d(1, 1, 1)
    with pytest.raises(RuntimeError, match="device_transform"):
        pkg.train.epoch_training([], model, None, None, epoch=0, n_gpus=None, device_transform=aug.Compose([]))


# ------------------------------------------------------------------------------------------------ the oracle itself
def _loop(x: np.ndarray, affine: np.ndarray, padding: str, nearest: bool) -> np.ndarray:
    """grid_sample(align_corners=False) restated voxel by voxel on index coordinates."""
    n, c, D, H, W = x.shape
    size = (D, H, W)
    out = np.zeros(x.shape, dtype=np.float64)
    for i in range(n):
        for d in range(D):
            for h in range(H):
                for w in range(W):
                    s = affine[i, :, :3] @ np.array([d, h, w], dtype=np.float64) + affine[i, :, 3]
                    if padding == "border":
                        s = np.clip(s, 0, np.array(size) - 1)
                    if nearest:
                        r = np.rint(s).astype(int)
                        if all(0 <= r[k] < size[k] for k in range(3)):
                            out[i, :, d, h, w] = x[i, :, r[0], r[1], r[2]]
                        continue
                    f = np.floor(s).astype(int)
                    t = s - f
                    acc = np.zeros(c)
                    for cd in (0, 1):
                        for ch in (0, 1):
                            for cw in (0, 1):
                                idx = (f[0] + cd, f[1] + ch, f[2] + cw)
                                wt = (t[0] if cd else 1 - t[0]) * (t[1] if ch else 1 - t[1]) * (t[2] if cw else 1 - t[2])
                                if all(0 <= idx[k] < size[k] for k in range(3)):
                                    acc += wt * x[i, :, idx[0], idx[1], idx[2]]
                    out[i, :, d, h, w] = acc
    return out


@pytest.mark.parametrize("padding", ["border", "zeros"])
def test_oracle_matches_an_explicit_loop(aug, padding):
    shape = (2, 2, 5, 6, 7)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(shape, generator=g, dtype=torch.float64)
    lab = (torch.rand(shape, generator=g) * 4).to(torch.uint8)
    keys = ("image", "label")
    comp = aug.Compose([aug.RandFlipd(keys, prob=1.0, spatial_axis=1),
                        aug.RandRotated(keys, range_x=0.6, range_y=0.5, range_z=0.7, prob=1.0, padding_mode=padding)])
    comp.set_random_state(2)
    p = comp.draw(2, 2, shape[2:])
    affine = p["affine"].numpy().copy()
    affine[:, :, 3] += np.array([0.3, -0.8, 0.45])                     # also sample past the boundary
    a = torch.from_numpy(affine)
    got = augment_oracle.resample(x, a, padding, "bilinear").numpy()
    assert np.abs(got - _loop(x.numpy(), affine, padding, False)).max() < 1e-12
    got_l = augment_oracle.resample(lab, a, padding, "nearest").numpy()
    assert np.array_equal(got_l, _loop(lab.numpy().astype(np.float64), affine, padding, True))
    # z-score and (a, b): channel-wise statistics of the resampled image, population std
    y = augment_oracle.intensity(torch.from_numpy(got), {"nonzero": False, "channel_wise": True},
                                 torch.tensor([[[2.0, 1.0], [1.0, 0.0]]] * 2, dtype=torch.float64)).numpy()
    z = (got[0, 0] - got[0, 0].mean()) / got[0, 0].std()
    assert np.abs(y[0, 0] - (2 * z + 1)).max() < 1e-12
