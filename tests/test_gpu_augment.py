"""Device augmentation (``augment.py``, ``csrc/augment.cu``) against the fp64 oracle (tests/augment_oracle.py) for the
parameters each batch drew: trilinear image and nearest label resample in both padding modes, flips bit for bit, the
z-score statistics, the fused intensity pass, run-to-run bit identity, and the training loop hook."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import augment_oracle  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
KEYS = ("image", "label")
SHAPES = [((2, 4, 24, 40, 33), 1), ((2, 4, 128, 128, 128), 3)]    # (image shape, label channels)


def _data(shape, n_labels, seed=0, zeros=0.0, scale=None, shift=None):
    """N(0, 1) image (times scale plus shift per channel), then a share ``zeros`` of exact zeros in every channel"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g)
    if scale is not None:
        x = x * torch.tensor(scale)[None, :, None, None, None] + torch.tensor(shift)[None, :, None, None, None]
    if zeros:
        x[torch.rand(shape, generator=g) < zeros] = 0.0
    lab = (torch.rand((shape[0], n_labels) + shape[2:], generator=g) * 4).to(torch.uint8)
    return x, lab


def _spatial(aug, padding="border", prob=0.5):
    return [aug.RandFlipd(KEYS, prob=prob, spatial_axis=0), aug.RandFlipd(KEYS, prob=prob, spatial_axis=1),
            aug.RandRotated(KEYS, range_x=0.2, range_y=0.2, range_z=0.2, prob=prob, padding_mode=padding)]


def _seed_with_mixed_rotation(comp, n, c, spatial):
    """a seed whose batch has samples with and without the rotation"""
    for s in range(1000):
        comp.set_random_state(s)
        done = [r[2]["do"] for r in comp.draw(n, c, spatial)["transforms"]]
        if any(done) and not all(done):
            comp.set_random_state(s)
            return s
    raise AssertionError("no seed mixes rotated and unrotated samples")


def _label_ties(params, spatial, band=1e-4):
    """voxels whose fp64 source coordinate lies within ``band`` voxels of a rounding tie on some axis.  The kernel's fp32
    coordinate is off by about extent * 2^-24 (measured below 1e-5 voxels at 128^3), so 1e-4 leaves a tenfold margin; the
    share of tie voxels grows with the band (3 axes * 2 * band per rotated voxel)."""
    src = augment_oracle.source_coordinates(params["affine"], spatial)
    if params["padding_mode"] == "border":
        src = torch.minimum(src.clamp(min=0), torch.tensor(spatial, dtype=torch.float64) - 1)
    return ((src - src.floor() - 0.5).abs() < band).any(-1)


@pytest.mark.parametrize("padding", ["border", "zeros"])
@pytest.mark.parametrize("shape,n_labels", SHAPES)
def test_resample_matches_fp64_oracle(pkg, shape, n_labels, padding):
    aug = pkg.augment
    comp = aug.Compose(_spatial(aug, padding))
    _seed_with_mixed_rotation(comp, shape[0], shape[1], shape[2:])
    x, lab = _data(shape, n_labels)
    out = comp({"image": x.to(DEV), "label": lab.to(DEV)})
    p = comp.last_params
    assert out["image"].shape == x.shape and out["label"].shape == lab.shape and out["label"].dtype == torch.uint8
    ref, ref_l = augment_oracle.augment(x, lab, p)
    got = out["image"].cpu().double()
    err = (got - ref).abs().max().item()
    rel = ((got - ref).norm() / ref.norm()).item()
    print("resample %s %s: max abs %.3e, rel-L2 %.3e" % (shape, padding, err, rel))
    # measured on an H100: at most 7.5e-5 and 4.2e-6 at 128^3
    assert err <= 1.5e-4 and rel <= 1e-5
    tie = _label_ties(p, shape[2:])[:, None].expand_as(ref_l)
    mism = out["label"].cpu().double() != ref_l
    assert not (mism & ~tie).any()
    assert tie.double().mean().item() < 1e-3


def _same_bits(a, b):
    """bit for bit, with every NaN counted as one value (the GPU returns its canonical NaN, not the payload it read)"""
    na, nb = a.isnan(), b.isnan()
    return torch.equal(na, nb) and torch.equal(a.masked_fill(na, 0.0).contiguous().view(torch.int32),
                                               b.masked_fill(nb, 0.0).contiguous().view(torch.int32))


def test_flips_and_prob_zero_are_bit_identical(pkg):
    aug = pkg.augment
    x, lab = _data((2, 3, 24, 40, 33), 2, seed=1)
    # signed zeros and non-finite values are copied as they are, and do not leak into their neighbours
    x[0, 0, 3, 4, 5], x[0, 1, 7, 8, 9], x[1, 2, 23, 39, 32], x[1, 0, 0, 0, 0] = -0.0, float("inf"), float("-inf"), float("nan")
    x[1, 1, 10, 11:20, 12] = -0.0
    xd, ld = x.to(DEV), lab.to(DEV)
    for axes in ((0,), (1,), (2,), (0, 2), None):
        for padding in ("border", "zeros"):
            comp = aug.Compose([aug.RandFlipd(KEYS, prob=1.0, spatial_axis=axes),
                                aug.RandRotated(KEYS, range_x=0.3, prob=0.0, padding_mode=padding)])
            out = comp({"image": xd, "label": ld})
            dims = [2 + a for a in (axes if axes is not None else (0, 1, 2))]
            assert _same_bits(out["image"], torch.flip(xd, dims)) and torch.equal(out["label"], torch.flip(ld, dims))
    comp = aug.Compose(_spatial(aug, prob=0.0) + [aug.RandScaleIntensityd("image", factors=0.1, prob=0.0),
                                                  aug.RandShiftIntensityd("image", offsets=0.1, prob=0.0)])
    out = comp({"image": xd, "label": ld, "other": 7})
    assert _same_bits(out["image"], xd) and torch.equal(out["label"], ld) and out["other"] == 7
    one = aug.RandFlipd(KEYS, prob=1.0, spatial_axis=1)({"image": xd[0], "label": ld[0]})      # one unbatched sample
    assert _same_bits(one["image"], torch.flip(xd[0], [2])) and torch.equal(one["label"], torch.flip(ld[0], [2]))


@pytest.mark.parametrize("nonzero", [False, True])
@pytest.mark.parametrize("channel_wise", [False, True])
def test_zscore_statistics_and_intensity_pass(pkg, nonzero, channel_wise):
    aug = pkg.augment
    shape = (2, 4, 24, 40, 33)
    x, lab = _data(shape, 1, seed=2, zeros=0.3, scale=[1.0, 3.0, 0.5, 2.0], shift=[0.0, 5.0, -1.0, 0.25])
    assert all(float((x[:, c] == 0).double().mean()) > 0.25 for c in range(4))       # every channel exercises `nonzero`
    # identity resample: the statistics are of the input itself
    comp = aug.Compose([aug.NormalizeIntensityd("image", nonzero=nonzero, channel_wise=channel_wise)])
    out = comp({"image": x.to(DEV)})
    st = comp.last_stats.cpu()
    xd = x.double()
    sel = (xd != 0) if nonzero else torch.ones_like(xd, dtype=torch.bool)
    ref = torch.stack([(xd * sel).sum((2, 3, 4)), (xd * xd * sel).sum((2, 3, 4)), sel.double().sum((2, 3, 4))], -1)
    assert torch.equal(st[..., 2], ref[..., 2])
    assert torch.allclose(st[..., :2], ref[..., :2], rtol=1e-13, atol=1e-9)
    p = comp.last_params
    y = augment_oracle.intensity(xd, p["normalize"], p["coef"])
    assert (out["image"].cpu().double() - y).abs().max().item() < 2e-6 * max(1.0, y.abs().max().item())
    # with a rotation, scale and shift in the same call
    comp = aug.Compose(_spatial(aug) + [aug.NormalizeIntensityd("image", nonzero=nonzero, channel_wise=channel_wise),
                                        aug.RandScaleIntensityd("image", factors=0.1, prob=1.0, channel_wise=True),
                                        aug.RandShiftIntensityd("image", offsets=0.1, prob=1.0)])
    _seed_with_mixed_rotation(comp, shape[0], shape[1], shape[2:])
    out = comp({"image": x.to(DEV), "label": lab.to(DEV)})
    ref, _ = augment_oracle.augment(x, None, comp.last_params)
    got = out["image"].cpu().double()
    err = (got - ref).abs().max().item()
    rel = ((got - ref).norm() / ref.norm()).item()
    print("full pipeline nonzero=%s channel_wise=%s: max abs %.3e, rel-L2 %.3e" % (nonzero, channel_wise, err, rel))
    # measured on an H100: at most 3.3e-5 and 2.2e-6
    assert err <= 1e-4 and rel <= 1e-5


def test_same_seed_is_bit_identical(pkg):
    aug = pkg.augment
    x, lab = _data((2, 4, 128, 128, 128), 3, seed=3)
    xd, ld = x.to(DEV), lab.to(DEV)
    comp, _ = aug.build_device_transform({"normalization_kwargs": {"channel_wise": True}, "training": {
        "spatial_augmentations": [{"name": "RandFlipD", "spatial_axis": 0, "prob": 0.5},
                                  {"name": "RandRotateD", "prob": 1.0, "range_x": 0.2, "range_y": 0.2, "range_z": 0.2}],
        "intensity_augmentations": [{"name": "RandScaleIntensityD", "factors": 0.1, "prob": 1.0},
                                    {"name": "RandShiftIntensityD", "offsets": 0.1, "prob": 1.0}]}})
    a = comp.set_random_state(11)({"image": xd, "label": ld})
    b = comp.set_random_state(11)({"image": xd, "label": ld})
    assert torch.equal(a["image"], b["image"]) and torch.equal(a["label"], b["label"])
    c = comp({"image": xd, "label": ld})                                         # next draws: a different batch
    assert not torch.equal(a["image"], c["image"])


KW = dict(n_features=4, n_outputs=3, base_width=8, encoder_blocks=[1, 1, 1], decoder_blocks=[1, 1, 1], dropout=0.0)


def _loader(n=3):
    out = []
    for i in range(n):
        g = torch.Generator().manual_seed(100 + i)
        out.append({"image": torch.randn(2, 4, 32, 32, 32, generator=g).pin_memory(),
                    "label": (torch.rand(2, 3, 32, 32, 32, generator=g) > 0.6).to(torch.uint8).pin_memory()})
    return out


def _train(pkg, sd, transform, graph):
    model = pkg.UNet3D(precision="bf16", deterministic=True, **KW).to(DEV)
    model.load_state_dict(sd)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    avg = pkg.train.epoch_training(_loader(), model, pkg.DiceLoss(sigmoid=True), opt, epoch=0, n_gpus=1, print_frequency=0,
                                   use_cuda_graph=graph, device_transform=transform)
    torch.cuda.synchronize()
    return avg, [p.detach().clone() for p in model.parameters()]


@pytest.mark.parametrize("graph", [False, True])
def test_epoch_training_with_device_transform(pkg, graph):
    aug = pkg.augment
    torch.manual_seed(0)
    sd = {k: v.clone() for k, v in pkg.UNet3D(**KW).state_dict().items()}
    full = aug.Compose(_spatial(aug, prob=1.0) + [aug.NormalizeIntensityd("image", channel_wise=True),
                                                  aug.RandScaleIntensityd("image", factors=0.1, prob=1.0),
                                                  aug.RandShiftIntensityd("image", offsets=0.1, prob=1.0)]).set_random_state(0)
    avg, params = _train(pkg, sd, full, graph)
    assert np.isfinite(avg) and 0.0 < avg < 1.0
    assert all(torch.isfinite(p).all() for p in params)
    # every prob = 0 and no intensity transform: the same losses and weights as without the transform, bit for bit
    avg0, params0 = _train(pkg, sd, aug.Compose(_spatial(aug, prob=0.0)), graph)
    avg1, params1 = _train(pkg, sd, None, graph)
    assert avg0 == avg1
    assert all(torch.equal(a, b) for a, b in zip(params0, params1))


def test_intensity_pass_on_an_unaligned_image(pkg):
    """b200unet_augment_intensity takes any float-aligned image pointer: an image starting 4 bytes past a 16-byte boundary
    (d*h*w a multiple of 4) gives the same values as an aligned one"""
    lib = pkg.lib.load_library()
    n, c, s = 2, 3, 16 * 20 * 24
    x = torch.randn(n, c, s, generator=torch.Generator().manual_seed(7)).to(DEV)
    coef = torch.tensor([1.5, -0.25] * (n * c), dtype=torch.float32, device=DEV)
    scratch = torch.empty(int(lib.b200unet_augment_scratch_bytes(n, c, s)), dtype=torch.uint8, device=DEV)
    outs = []
    for shift in (0, 1):
        buf = torch.empty(n * c * s + 4, device=DEV)
        img = buf[shift:shift + n * c * s]
        img.copy_(x.reshape(-1))
        pkg.lib.check(lib.b200unet_augment_intensity(img.data_ptr(), n, c, s, 0, 0, 0, coef.data_ptr(), scratch.data_ptr(),
                                                     pkg.lib.stream_ptr()), "augment_intensity")
        outs.append(img.clone())
    assert torch.equal(outs[0], outs[1])                           # fmaf(x, a, b) on both paths
    assert torch.allclose(outs[0], x.reshape(-1) * 1.5 - 0.25, rtol=1e-6, atol=1e-6)
