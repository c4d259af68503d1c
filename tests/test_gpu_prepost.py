"""The steps before / after the path on the device (SURVEY.md section 8f rows 2 and 4), through the C ABI, against
the pinned oracle restatements and the committed reference fixtures: sliding-window tiling kernels, one-hot targets,
z-score normalisation, activation + threshold -> label map; plus the step-loop pieces around the path (CUDA-graph
replayed training step, forward-only plans, the one-outstanding-forward guard, soft Dice targets)."""
import os
import sys

import numpy as np
import pytest
import torch
from torch import nn

from oracle import UNetConfig, make_state_dict, unet3d_forward, dice_loss, sliding_window_inference
from oracle.prepost_oracle import one_hot_encode, label_map_from_one_hot, normalize_intensity

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)
from recipe_prepost import ONE_HOT_CASES, LABEL_MAP_CASES, label_map_input, prediction_input  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = np.load(os.path.join(HERE, "golden", "prepost.npz"))


# ------------------------------------------------------------------------------------------------ sliding window
@pytest.mark.parametrize("mode", ["constant", "gaussian"])
@pytest.mark.parametrize("shape,roi,swb", [((2, 2, 20, 24, 28), (16, 16, 16), 4), ((1, 3, 33, 17, 40), (16, 16, 24), 5),
                                           ((1, 1, 12, 40, 12), (16, 16, 16), 1)])
def test_tiling_kernels_match_oracle_inferer(pkg, mode, shape, roi, swb):
    torch.manual_seed(0)
    net = nn.Conv3d(shape[1], 3, kernel_size=3, padding=1)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(0))
    inf = pkg.predict.SlidingWindowInferer(roi_size=roi, sw_batch_size=swb, overlap=0.25, mode=mode)
    with torch.no_grad():
        ref = sliding_window_inference(x, roi, net, overlap=0.25, mode=mode)
        netd = net.to(DEV)
        got = inf(x.to(DEV), netd)
        again = inf(x.to(DEV), netd)
    assert got.shape == ref.shape
    assert float((got.cpu() - ref).abs().max()) < 1e-4 * max(1.0, float(ref.abs().max()))
    assert torch.equal(got, again)                                   # tile-ordered accumulation: bit-reproducible


def test_inferer_rejects_gradient_tracking_network(pkg):
    net = nn.Conv3d(1, 1, 1).to(DEV)
    inf = pkg.predict.SlidingWindowInferer(roi_size=(8, 8, 8))
    with pytest.raises(RuntimeError, match="inference-only"):
        inf(torch.zeros(1, 1, 12, 12, 12, device=DEV), net)


def test_inferer_identity_property_monai_cases(pkg):
    """MONAI's own sliding-window unit test: ``compute = data + 1`` must return ``inputs + 1`` for every tiling."""
    from test_oracle_monai_cases import MONAI_SW_CASES
    for shape, roi, swb, overlap, mode in MONAI_SW_CASES:
        x = torch.randn(shape, generator=torch.Generator().manual_seed(0)).to(DEV)
        inf = pkg.predict.SlidingWindowInferer(roi_size=roi, sw_batch_size=swb, overlap=overlap, mode=mode)
        with torch.no_grad():
            out = inf(x, lambda data: data + 1)
        assert float((out - (x + 1)).abs().max()) < 1e-4, (shape, roi, mode)


def test_dice_kernel_reproduces_monai_published_values(pkg):
    from test_oracle_monai_cases import MONAI_DICE_CASES
    for kw, x, t, expected in MONAI_DICE_CASES:
        loss = pkg.DiceLoss(**kw)(x.to(DEV), t.to(DEV))
        assert abs(float(loss) - expected) < 2e-6, kw


# ------------------------------------------------------------------------------------------------ one-hot / label map / z-score
@pytest.mark.parametrize("name", sorted(ONE_HOT_CASES))
def test_one_hot_kernel_matches_reference_fixture(pkg, name):
    shape, values, n_labels, labels, seed = ONE_HOT_CASES[name]
    data = label_map_input(shape, values, seed)
    got = pkg.prepost.compile_one_hot_encoding(data.to(DEV), n_labels=n_labels, labels=labels, return_4d=False).cpu().numpy()
    shp = tuple(int(v) for v in GOLD["one_hot_shape::" + name])
    ref = np.unpackbits(GOLD["one_hot::" + name])[: int(np.prod(shp))].reshape(shp)
    assert got.dtype == np.uint8 and got.shape == shp
    assert (got == ref).all()                                                   # bit-exact vs the unmodified reference
    assert (got == one_hot_encode(data.numpy(), n_labels, labels)).all()


def test_one_hot_full_size_properties(pkg):
    """BraTS-sized label map (128^3): every voxel's channels follow the hierarchy WT >= TC >= ET, counts match torch."""
    g = torch.Generator().manual_seed(5)
    lab = torch.tensor([0.0, 1.0, 2.0, 4.0])[torch.randint(0, 4, (1, 1, 128, 128, 128), generator=g)].to(DEV)
    y = pkg.prepost.compile_one_hot_encoding(lab, n_labels=3, labels=[[1, 2, 4], [1, 4], 4], return_4d=False)
    assert int(y[0, 0].sum()) == int((lab != 0).sum()) and int(y[0, 2].sum()) == int((lab == 4).sum())
    assert bool((y[0, 0] >= y[0, 1]).all()) and bool((y[0, 1] >= y[0, 2]).all())


@pytest.mark.parametrize("name", sorted(LABEL_MAP_CASES))
def test_label_map_kernel_matches_reference_fixture(pkg, name):
    shape, labels, kw, seed = LABEL_MAP_CASES[name]
    p = prediction_input(shape, seed)
    got = pkg.prepost.convert_one_hot_to_label_map(p.to(DEV), labels=labels, **kw).cpu().numpy()
    ref = GOLD["label_map::" + name]
    assert got.dtype == np.int16 and got.shape == ref.shape
    assert (got == ref).all()


def test_label_map_fused_activation(pkg):
    logits = torch.randn(3, 10, 11, 12, generator=torch.Generator().manual_seed(7)) * 3
    for act, fn in (("sigmoid", torch.sigmoid), ("softmax", lambda z: torch.softmax(z, dim=0))):
        for kw in (dict(label_hierarchy=True), dict(), dict(sum_then_threshold=True, threshold=0.7)):
            got = pkg.prepost.convert_one_hot_to_label_map(logits.to(DEV), [2, 1, 4], activation=act, **kw).cpu().numpy()
            ref = label_map_from_one_hot(fn(logits).numpy(), [2, 1, 4], **kw)
            assert (got != ref).mean() < 1e-3                                   # ties at the threshold: exp rounding only


@pytest.mark.parametrize("nonzero,channel_wise", [(False, False), (True, False), (False, True), (True, True)])
def test_zscore_kernel_matches_oracle_unpinned(pkg, nonzero, channel_wise):
    g = torch.Generator().manual_seed(9)
    x = torch.randn(4, 20, 24, 28, generator=g) * torch.tensor([1.0, 5.0, 0.1, 30.0]).view(4, 1, 1, 1) + 3.0
    x[:, :5] = 0.0                                                               # background voxels for `nonzero`
    got = pkg.prepost.normalize_intensity(x.to(DEV), nonzero=nonzero, channel_wise=channel_wise).cpu().numpy()
    ref = normalize_intensity(x.numpy(), nonzero=nonzero, channel_wise=channel_wise)
    assert np.abs(got - ref).max() < 1e-4


# ------------------------------------------------------------------------------------------------ step loop around the path
KW = dict(n_features=2, n_outputs=2, base_width=8, encoder_blocks=[1, 1, 1], decoder_blocks=[1, 1, 1])


def _batch(seed, shape=(2, 2, 16, 16, 16)):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g)
    t = (torch.rand((shape[0], KW["n_outputs"]) + shape[2:], generator=g) > 0.6).to(torch.uint8)
    return x, t


def test_graphed_train_step_matches_eager(pkg):
    """GraphedTrainStep (captured forward + Dice + backward, flat gradient bucket, eager fused Adam) must produce the same
    losses and the same parameters as the eager loop over the same batches (dropout disabled to share the arithmetic)."""
    sd = make_state_dict(UNetConfig(**KW), seed=3)
    runs = {}
    for mode in ("eager", "graph"):
        torch.manual_seed(0)
        model = pkg.UNet3D(precision="split", dropout=0.0, **KW).to(DEV)
        model.load_state_dict(sd)
        model.train()
        crit = pkg.DiceLoss(sigmoid=True)
        opt = torch.optim.Adam(model.parameters(), lr=1e-3)
        losses = []
        step = pkg.train.GraphedTrainStep(model, crit, opt, (2, 2, 16, 16, 16), (2, 2, 16, 16, 16)) if mode == "graph" else None
        for i in range(4):
            x, t = _batch(100 + i)
            if step is not None:
                losses.append(float(step(x.pin_memory(), t.pin_memory()).item()))
            else:
                opt.zero_grad()
                loss = crit(model(x.to(DEV)), t.to(DEV))
                loss.backward()
                opt.step()
                losses.append(float(loss.item()))
        runs[mode] = (losses, [p.detach().clone() for p in model.ordered_parameters()])
        if mode == "graph":
            assert model.flat_gradient_bucket() is not None
            lo = model.flat_gradient_bucket().data_ptr()
            assert all(lo <= p.grad.data_ptr() < lo + 4 * model.flat_gradient_bucket().numel() for p in model.parameters())
    for a, b in zip(runs["eager"][0], runs["graph"][0]):
        assert abs(a - b) < 1e-5
    num = sum(float((a - b).double().pow(2).sum()) for a, b in zip(runs["eager"][1], runs["graph"][1])) ** 0.5
    den = sum(float(a.double().pow(2).sum()) for a in runs["eager"][1]) ** 0.5
    assert num / den < 1e-4


@pytest.mark.parametrize("arch", ["unet3d", "unet3d_convT", "dynunet"])
def test_deterministic_backward_repeats_bit_for_bit(pkg, arch):
    """A deterministic plan's backward writes the same flat gradient bucket bit for bit every time, and writes all of it (unet3d_convT:
    the transposed-convolution up-sampling, whose bias gradient sums 32^3 voxels over a full grid of blocks)."""
    torch.manual_seed(0)
    if arch.startswith("unet3d"):
        model = pkg.UNet3D(precision="bf16", deterministic=True, dropout=0.0, n_features=2, n_outputs=2, base_width=8,
                           use_transposed_convolutions=arch == "unet3d_convT").to(DEV)
        shape, tshape = (2, 2, 32, 32, 32), (2, 2, 32, 32, 32)
    else:
        model = pkg.DynUNet(spatial_dims=3, in_channels=2, out_channels=2, kernel_size=[[3, 3, 3]] * 4, strides=[[1, 1, 1]] + [[2, 2, 2]] * 3,
                            upsample_kernel_size=[[2, 2, 2]] * 3, filters=[8, 16, 24, 32], precision="bf16", deterministic=True).to(DEV)
        shape, tshape = (2, 2, 32, 32, 32), (2, 2, 32, 32, 32)
    model.train()
    crit = pkg.DiceLoss(sigmoid=True)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(shape, generator=g).to(DEV)
    t = (torch.rand(tshape, generator=g) > 0.6).to(torch.uint8).to(DEV)
    model.use_flat_gradients(True)
    # whole backward
    crit(model(x), t).backward()
    torch.cuda.synchronize()
    whole = model.flat_gradient_bucket().clone()
    for p in model.parameters():
        p.grad = None
    crit(model(x), t).backward()
    torch.cuda.synchronize()
    assert torch.equal(model.flat_gradient_bucket(), whole), "a deterministic plan must repeat its gradients bit for bit"
    # poison the bucket first so that a gradient nobody writes shows up
    for p in model.parameters():
        p.grad = None
    model.flat_gradient_bucket().fill_(float("nan"))
    crit(model(x), t).backward()
    torch.cuda.synchronize()
    assert torch.equal(model.flat_gradient_bucket(), whole)


def test_epoch_training_with_cuda_graph_and_short_last_batch(pkg):
    torch.manual_seed(0)
    model = pkg.UNet3D(precision="bf16", **KW).to(DEV)
    crit = pkg.DiceLoss(sigmoid=True)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    loader = []
    for i in range(3):
        x, t = _batch(i)
        loader.append({"image": x, "label": t})
    x, t = _batch(9, shape=(1, 2, 16, 16, 16))                                   # short last batch -> eager fallback
    loader.append({"image": x, "label": t})
    before = [p.detach().clone() for p in model.parameters()]
    avg = pkg.train.epoch_training(loader, model, crit, opt, epoch=0, n_gpus=1, print_frequency=0, use_cuda_graph=True)
    assert 0.0 < avg < 1.0
    assert all(not torch.equal(a, b) for a, b in zip(before, model.parameters()) if a.numel() > 8)


@pytest.mark.parametrize("precision", ["bf16", "split"])
def test_deterministic_mode_gives_bit_identical_gradients(pkg, precision):
    """deterministic=True: the split-K weight gradients go through per-split partial sums + a fixed-order reduction (no fp32
    atomics); two backward passes on the same inputs must agree BIT FOR BIT, and agree with the default (atomic) mode to
    rounding.  Shapes large enough that every weight-gradient kernel splits K over several CTAs."""
    kw = dict(n_features=4, n_outputs=3, base_width=16)
    sd = make_state_dict(UNetConfig(**kw), seed=9)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 4, 64, 64, 64, generator=g).to(DEV)
    t = (torch.rand(2, 3, 64, 64, 64, generator=g) > 0.7).to(torch.uint8).to(DEV)
    grads = {}
    for det in (True, False):
        model = pkg.UNet3D(precision=precision, deterministic=det, **kw).to(DEV)
        model.load_state_dict(sd)
        model.train()
        model.set_dropout_scale(torch.ones(2, 16))
        runs = []
        for _ in range(2):
            model.zero_grad(set_to_none=True)
            pkg.DiceLoss(sigmoid=True)(model(x), t).backward()
            runs.append([p.grad.clone() for p in model.ordered_parameters()])
        if det:
            for k, a, b in zip(model._keys, runs[0], runs[1]):
                assert torch.equal(a, b), k
        grads[det] = runs[0]
    num = sum(float((a - b).double().pow(2).sum()) for a, b in zip(grads[True], grads[False])) ** 0.5
    den = sum(float(b.double().pow(2).sum()) for b in grads[False]) ** 0.5
    assert num / den < 1e-4


def test_second_forward_before_backward_raises(pkg):
    model = pkg.UNet3D(precision="bf16", **KW).to(DEV).train()
    x1, _ = _batch(1)
    x2, _ = _batch(2)
    o1 = model(x1.to(DEV))
    o2 = model(x2.to(DEV))
    o2.sum().backward()                                                          # the latest forward is fine
    with pytest.raises(RuntimeError, match="overwritten the saved activations"):
        o1.sum().backward()
    # an eval / no_grad forward in between uses its own forward-only plan and does not disturb the training one
    o3 = model(x1.to(DEV))
    with torch.no_grad():
        model(x2.to(DEV))
    o3.sum().backward()


def test_forward_only_plan_matches_training_plan_and_is_smaller(pkg):
    kw = dict(n_features=1, n_outputs=1, base_width=8, encoder_blocks=[1, 2, 2, 2, 2])
    sd = make_state_dict(UNetConfig(**kw), seed=6)
    model = pkg.UNet3D(precision="split", **kw).to(DEV)
    model.load_state_dict(sd)
    model.eval()
    x = torch.randn(2, 1, 32, 48, 32, device=DEV)
    with torch.no_grad():
        y_inf = model(x)
    y_train_plan = model(x)                                                       # grad enabled: training plan, eval math
    assert torch.equal(y_inf, y_train_plan.detach())
    plans = {k[-1]: p for k, p in model._plans.items()}
    assert plans[True].ws_bytes < 0.5 * plans[False].ws_bytes
    sd64 = {k: v.double() for k, v in sd.items()}
    ref = unet3d_forward(sd64, x.double().cpu(), UNetConfig(**kw))
    assert float((y_inf.double().cpu() - ref).norm() / ref.norm()) < 1e-3
    with pytest.raises(RuntimeError):
        y_inf.sum().backward()


def test_forward_only_plan_repacks_weights_after_an_update(pkg):
    """forward-only plans keep their packed bf16 weights while no parameter changes (tiled inference); an in-place update
    (optimizer step, load_state_dict) must be picked up by the next forward."""
    kw = dict(n_features=2, n_outputs=2, base_width=8, encoder_blocks=[1, 1], decoder_blocks=[1, 1])
    model = pkg.UNet3D(precision="split", **kw).to(DEV).eval()
    x = torch.randn(1, 2, 16, 16, 16, device=DEV)
    with torch.no_grad():
        y0 = model(x)
        y1 = model(x)                                      # packed weights reused
        assert torch.equal(y0, y1)
        for p in model.parameters():
            p.mul_(1.5)                                    # bumps the version counters
        y2 = model(x)
        sd = {k: v / 1.5 for k, v in model.state_dict().items()}
        model.load_state_dict(sd)
        y3 = model(x)
    assert float((y2 - y0).abs().max()) > 1e-3
    assert float((y3 - y0).abs().max()) < 1e-4 * max(1.0, float(y0.abs().max()))


def test_dice_accepts_soft_float_targets(pkg):
    g = torch.Generator().manual_seed(4)
    logits = torch.randn(2, 3, 9, 10, 11, generator=g)
    soft = torch.rand(2, 3, 9, 10, 11, generator=g)                               # label-smoothed / interpolated target
    lg = logits.to(DEV).requires_grad_(True)
    loss = pkg.DiceLoss(sigmoid=True)(lg, soft.to(DEV))
    loss.backward()
    lr = logits.double().requires_grad_(True)
    ref = dice_loss(lr, soft.double())
    ref.backward()
    assert abs(float(loss) - float(ref)) < 1e-6
    assert float((lg.grad.double().cpu() - lr.grad).norm() / lr.grad.norm()) < 1e-5
    hard = (soft > 0.5)
    l_bool = pkg.DiceLoss(sigmoid=True)(lg.detach(), hard.to(DEV))                # bool -> uint8 path
    assert abs(float(l_bool) - float(dice_loss(logits.double(), hard.double()))) < 1e-6
