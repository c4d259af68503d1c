"""Many-class heads (9..128 outputs) on the GPU: the tensor-core head kernels through the C ABI against fp64 einsum, UNet3D
in split precision against the reference's multi-class fixture (tests/golden/multiclass.npz), bf16 against torch's own bf16
autocast, DynUNet with its bias, a cross-entropy step, and the existing machinery (launch count, two-part backward,
determinism, input-gradient plans, CUDA graphs, sliding windows, pre/post-processing) at 104 classes."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import UNetConfig, make_state_dict, unet3d_forward, dice_loss, sliding_window_inference
from oracle.dynunet_oracle import make_dynunet_state_dict, dynunet_forward
from oracle.prepost_oracle import one_hot_encode, label_map_from_one_hot

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from recipe import golden_inputs, dropout_mask  # noqa: E402
from make_golden_multiclass import (TRAIN_CASES, SOFTMAX_CASE, SHAPE, SUB8, HEAD, N_LABELS, LABEL_MAP_CASES,  # noqa: E402
                                    one_hot_input, label_map_prediction, labels)

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


def _cos(a, b):
    a, b = np.asarray(a, dtype=np.float64).ravel(), np.asarray(b, dtype=np.float64).ravel()
    return float((a * b).sum() / (np.linalg.norm(a) * np.linalg.norm(b) + 1e-300))


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "multiclass.npz"))


# ------------------------------------------------------------------------------------------------ kernels through the ABI
def _act_in(pkg, shape, c, split, seed):
    """an NDHWC activation whose value (hi + lo) is known exactly in fp64"""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(shape + (c,), generator=g)
    hi = v.to(torch.bfloat16)
    lo = (v - hi.float()).to(torch.bfloat16) if split else None
    val = hi.double() + (lo.double() if split else 0)
    return pkg.lib.Act(hi.to(DEV).contiguous(), lo.to(DEV).contiguous() if split else None), val


def _act_value(a):
    return a.hi.double().cpu() + (a.lo.double().cpu() if a.lo is not None else 0)


def _head_case(pkg, n_out, c, split, shape, act=0, seed=0):
    L = pkg.lib
    x, xv = _act_in(pkg, shape, c, split, seed)
    g = torch.Generator().manual_seed(seed + 1)
    w = (torch.randn(n_out, c, generator=g) / c ** 0.5)
    logits = torch.empty((shape[0], n_out) + shape[1:], device=DEV)
    L.head_fwd(x, w.to(DEV), n_out, act, logits)
    ref = torch.einsum("ndhwc,oc->nodhw", xv, w.double())
    if act == 1:
        ref = torch.sigmoid(ref)
    elif act == 2:
        ref = torch.softmax(ref, dim=1)
    return x, xv, w, logits, ref


HEAD_SHAPES = [(n_out, c) for n_out in (9, 16, 24, 104, 128) for c in (8, 32, 48, 64)]


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("n_out,c", HEAD_SHAPES)
def test_head_kernels_match_fp64_einsum(pkg, n_out, c, split):
    shape = (2, 8, 9, 10)                                             # 1440 voxels: 12 tiles, the last one partial
    x, xv, w, logits, ref = _head_case(pkg, n_out, c, split, shape)
    tol = 2e-5 if split else 1e-2
    assert _rel(logits, ref) < tol
    # backward: dx = g w, dw = sum_v g x
    L = pkg.lib
    gl = torch.randn(logits.shape, generator=torch.Generator().manual_seed(7))
    dx = L.Act.empty(*shape, c, split=split)
    dw = torch.empty(n_out, c, device=DEV)
    L.head_bwd(x, w.to(DEV), n_out, gl.to(DEV), dx, dw)
    torch.cuda.synchronize()
    ref_dx = torch.einsum("nodhw,oc->ndhwc", gl.double(), w.double())
    ref_dw = torch.einsum("nodhw,ndhwc->oc", gl.double(), xv)
    assert _rel(_act_value(dx), ref_dx) < (2e-5 if split else 1e-2)
    assert _rel(dw, ref_dw) < (2e-5 if split else 1e-2)
    # bit-identical on a second run
    dx2 = L.Act.empty(*shape, c, split=split)
    dw2 = torch.empty(n_out, c, device=DEV)
    L.head_bwd(x, w.to(DEV), n_out, gl.to(DEV), dx2, dw2)
    torch.cuda.synchronize()
    assert torch.equal(dw, dw2) and torch.equal(dx.hi, dx2.hi)
    assert not split or torch.equal(dx.lo, dx2.lo)


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("n_out", [9, 104])
def test_head_kernels_odd_extents_straddle_samples(pkg, n_out, split):
    shape = (2, 5, 7, 3)                                               # 105 voxels per sample: tiles straddle the samples
    c = 32
    x, xv, w, logits, ref = _head_case(pkg, n_out, c, split, shape, seed=3)
    assert _rel(logits, ref) < (2e-5 if split else 1e-2)
    L = pkg.lib
    gl = torch.randn(logits.shape, generator=torch.Generator().manual_seed(8))
    dx = L.Act.empty(*shape, c, split=split)
    dw = torch.empty(n_out, c, device=DEV)
    L.head_bwd(x, w.to(DEV), n_out, gl.to(DEV), dx, dw)
    torch.cuda.synchronize()
    assert _rel(_act_value(dx), torch.einsum("nodhw,oc->ndhwc", gl.double(), w.double())) < (2e-5 if split else 1e-2)
    assert _rel(dw, torch.einsum("nodhw,ndhwc->oc", gl.double(), xv)) < (2e-5 if split else 1e-2)


@pytest.mark.parametrize("act", [1, 2])
@pytest.mark.parametrize("n_out", [9, 24, 128])
def test_head_activation_epilogues(pkg, n_out, act):
    _, _, _, logits, ref = _head_case(pkg, n_out, 32, True, (2, 5, 7, 3), act=act, seed=5)
    assert float((logits.double().cpu() - ref).abs().max()) < 1e-5
    if act == 2:                                                       # pad channels excluded from the softmax
        assert float((logits.double().sum(dim=1) - 1).abs().max()) < 1e-5


def test_head_refuses_129_outputs_with_the_limit(pkg):
    L = pkg.lib
    x, _ = _act_in(pkg, (1, 4, 4, 4), 8, False, 0)
    with pytest.raises(RuntimeError, match=r"n_outputs=129 unsupported \(1\.\.128\)"):
        L.head_fwd(x, torch.zeros(129, 8, device=DEV), 129, 0, torch.empty(1, 129, 4, 4, 4, device=DEV))


# ------------------------------------------------------------------------------------------------ UNet3D against the reference
def _golden_model(pkg, kw, precision="split", **extra):
    cfg = UNetConfig(**kw)
    model = pkg.UNet3D(precision=precision, **extra, **kw).to(DEV)
    model.load_state_dict(make_state_dict(cfg, seed=0), strict=True)
    return cfg, model


def _golden_step(pkg, kw, precision="split", **extra):
    cfg, model = _golden_model(pkg, kw, precision, **extra)
    x, t, g3 = golden_inputs(SHAPE, cfg.n_outputs)
    model.train()
    model.set_dropout_scale(dropout_mask(SHAPE[0], cfg.enc_widths()[0], cfg.dropout, g3))
    out = model(x.to(DEV))
    loss = pkg.DiceLoss(sigmoid=True)(out, t.to(DEV))
    loss.backward()
    torch.cuda.synchronize()
    return model, out.detach().cpu(), float(loss)


@pytest.mark.parametrize("name", sorted(TRAIN_CASES))
def test_split_precision_matches_multiclass_fixture(pkg, gold, name):
    """north-star bounds: logits rel-L2 < 1e-3, |dDice| < 1e-3 relative, every gradient norm within 3 %, head gradient
    cosine > 0.999"""
    model, out, loss = _golden_step(pkg, TRAIN_CASES[name])
    rel = _rel(out[SUB8], gold[name + "::logits_sub8"])
    dice = float(gold[name + "::dice"])
    grads = dict(model.named_parameters())
    norms = np.array([float(grads[k].grad.double().norm()) for k in gold[name + "::grad_keys"]])
    ratio = norms / gold[name + "::grad_norms"]
    cos = _cos(grads[HEAD].grad.cpu().numpy(), gold[name + "::grad_head"])
    print("%s: logits rel-L2 %.3e, dDice %.3e, gradient-norm ratios %.4f..%.4f, head-gradient cosine %.6f"
          % (name, rel, abs(loss - dice), ratio.min(), ratio.max(), cos))
    assert rel < 1e-3
    assert abs(loss - dice) < 1e-3 * abs(dice)
    assert np.all(np.abs(ratio - 1) < 3e-2)
    assert cos > 0.999


def test_softmax_eval_forward_matches_fixture(pkg, gold):
    name, kw = SOFTMAX_CASE
    _, model = _golden_model(pkg, kw)
    model.eval()
    x, _, _ = golden_inputs(SHAPE, kw["n_outputs"])
    with torch.no_grad():
        p = model(x.to(DEV)).cpu()
    assert _rel(p[SUB8], gold[name + "::sub8"]) < 1e-3
    assert float((p.double().sum(dim=1) - 1).abs().max()) < 1e-5


def test_bf16_mode_is_torch_autocast_class_at_104_outputs(pkg):
    """bf16 mode rounds the head weights and dlogits to bf16; logits and the whole gradient stay within 1.25x the error
    of torch's bf16 autocast on the same graph"""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    kw = dict(n_features=4, n_outputs=104, base_width=16)
    cfg = UNetConfig(**kw)
    sd = make_state_dict(cfg, seed=0)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, 4, 32, 32, 32, generator=g)
    t = (torch.rand(1, 104, 32, 32, 32, generator=g) > 0.7).to(torch.uint8)

    def oracle(dtype, autocast):
        sdr = {k: v.to(DEV, dtype).requires_grad_(True) for k, v in sd.items()}
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            out = unet3d_forward(sdr, x.to(DEV, dtype), cfg)
        dice_loss(out.float() if autocast else out, t.to(DEV)).backward()
        return out.detach().double(), {k: v.grad.double() for k, v in sdr.items()}

    ref_out, ref_g = oracle(torch.float64, False)
    ac_out, ac_g = oracle(torch.float32, True)
    model = pkg.UNet3D(precision="bf16", **kw).to(DEV)
    model.load_state_dict(sd, strict=True)
    model.train()
    model.set_dropout_scale(torch.ones(1, 16))
    out = model(x.to(DEV))
    pkg.DiceLoss(sigmoid=True)(out, t.to(DEV)).backward()
    ours_g = {k: p.grad.double() for k, p in model.named_parameters()}

    def whole(gs):
        num = sum(float((gs[k] - ref_g[k]).pow(2).sum()) for k in ref_g)
        return (num / sum(float(v.pow(2).sum()) for v in ref_g.values())) ** 0.5
    e_out, a_out = _rel(out.detach(), ref_out), _rel(ac_out, ref_out)
    e_g, a_g = whole(ours_g), whole(ac_g)
    e_h, a_h = _rel(ours_g[HEAD], ref_g[HEAD]), _rel(ac_g[HEAD], ref_g[HEAD])
    print("bf16 vs autocast: logits %.3e / %.3e, whole gradient %.3e / %.3e, head gradient %.3e / %.3e"
          % (e_out, a_out, e_g, a_g, e_h, a_h))
    assert e_out <= 1.25 * a_out and e_g <= 1.25 * a_g
    assert e_h <= 2 * a_h + 5e-3


def _dynunet_kw(out_channels):
    return dict(spatial_dims=3, in_channels=4, out_channels=out_channels, kernel_size=[[3, 3, 3]] * 4,
                strides=[[1, 1, 1]] + [[2, 2, 2]] * 3, upsample_kernel_size=[[2, 2, 2]] * 3, filters=[16, 24, 32, 48])


def test_dynunet_14_outputs_matches_oracle_with_bias(pkg):
    kw = _dynunet_kw(14)
    sd = make_dynunet_state_dict(4, 14, kw["filters"], seed=0)
    sd["output_block.conv.conv.bias"] = torch.linspace(-0.5, 0.5, 14)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 4, 32, 32, 32, generator=g)
    t = (torch.rand(2, 14, 32, 32, 32, generator=g) > 0.7).to(torch.uint8)
    sd64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    ref = dynunet_forward(sd64, x.double(), 4)
    dice_loss(ref, t).backward()
    model = pkg.DynUNet(precision="split", **kw).to(DEV)
    model.load_state_dict(sd, strict=True)
    model.train()
    out = model(x.to(DEV))
    pkg.DiceLoss(sigmoid=True)(out, t.to(DEV)).backward()
    assert _rel(out.detach(), ref.detach()) < 1e-3
    for k, p in model.named_parameters():
        r = sd64[k].grad
        assert abs(float(p.grad.double().norm()) / float(r.norm()) - 1) < 3e-2, k
        if p.numel() >= 14:
            assert _cos(p.grad.cpu().numpy(), r.numpy()) > 0.999, k
    bias = model.output_block.conv.conv.bias.grad.double().cpu()
    assert _rel(bias, sd64["output_block.conv.conv.bias"].grad) < 1e-4


def test_cross_entropy_step_matches_oracle_autograd(pkg):
    """any dlogits feed the backward: CrossEntropyLoss on a label-map target"""
    kw = dict(n_features=4, n_outputs=24, base_width=8)
    cfg = UNetConfig(**kw)
    sd = make_state_dict(cfg, seed=1)
    g = torch.Generator().manual_seed(6)
    x = torch.randn(1, 4, 32, 32, 32, generator=g)
    lab = torch.randint(0, 24, (1, 32, 32, 32), generator=g)
    sd64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    torch.nn.CrossEntropyLoss()(unet3d_forward(sd64, x.double(), cfg, dropout_mask=torch.ones(1, 8)), lab).backward()
    model = pkg.UNet3D(precision="split", **kw).to(DEV)
    model.load_state_dict(sd, strict=True)
    model.train()
    model.set_dropout_scale(torch.ones(1, 8))
    torch.nn.CrossEntropyLoss()(model(x.to(DEV)), lab.to(DEV)).backward()
    for k, p in model.named_parameters():
        r = sd64[k].grad
        assert abs(float(p.grad.double().norm()) / float(r.norm()) - 1) < 3e-2, k
        assert _cos(p.grad.cpu().numpy(), r.numpy()) > 0.999, k


# ------------------------------------------------------------------------------------------------ machinery at 104 outputs
KW104 = dict(n_features=2, n_outputs=104, base_width=8)


def _batch(seed, shape=(2, 2, 32, 32, 32), n_out=104):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g)
    t = (torch.rand((shape[0], n_out) + shape[2:], generator=g) > 0.6).to(torch.uint8)
    return x, t


def test_104_outputs_take_the_launches_of_3_outputs(pkg):
    counts = {}
    for n_out in (3, 104):
        model = pkg.UNet3D(precision="bf16", n_features=2, n_outputs=n_out, base_width=8).to(DEV)
        model.train()
        x, t = _batch(1, n_out=n_out)
        pkg.DiceLoss(sigmoid=True)(model(x.to(DEV)), t.to(DEV)).backward()
        torch.cuda.synchronize()
        counts[n_out] = (model.launches_last_forward, model.launches_last_backward)
    assert counts[104][0] == counts[3][0]


@pytest.mark.parametrize("precision", ["bf16", "split"])
def test_two_part_and_deterministic_backward_at_104_outputs(pkg, precision):
    model = pkg.UNet3D(precision=precision, deterministic=True, dropout=0.0, **KW104).to(DEV)
    model.train()
    crit = pkg.DiceLoss(sigmoid=True)
    x, t = _batch(5)
    x, t = x.to(DEV), t.to(DEV)
    model.use_flat_gradients(True)
    crit(model(x), t).backward()
    torch.cuda.synchronize()
    whole = model.flat_gradient_bucket().clone()
    for p in model.parameters():
        p.grad = None
    crit(model(x), t).backward()
    torch.cuda.synchronize()
    assert torch.equal(model.flat_gradient_bucket(), whole)
    for p in model.parameters():
        p.grad = None
    model.flat_gradient_bucket().fill_(float("nan"))
    model._defer_backward_tail = True
    crit(model(x), t).backward()
    model._defer_backward_tail = False
    torch.cuda.synchronize()
    model.finish_backward()
    torch.cuda.synchronize()
    assert torch.equal(model.flat_gradient_bucket(), whole)


def test_non_deterministic_plan_head_gradient_is_reproducible(pkg):
    model = pkg.UNet3D(precision="bf16", dropout=0.0, **KW104).to(DEV)
    model.train()
    x, t = _batch(6)
    heads = []
    for _ in range(2):
        model.zero_grad(set_to_none=True)
        pkg.DiceLoss(sigmoid=True)(model(x.to(DEV)), t.to(DEV)).backward()
        heads.append(dict(model.named_parameters())[HEAD].grad.clone())
    assert torch.equal(heads[0], heads[1])


def test_input_grad_plan_keeps_parameter_gradients_bit_identical(pkg):
    sd = make_state_dict(UNetConfig(**KW104), seed=2)
    x, t = _batch(7)
    runs = {}
    for flagged in (False, True):
        model = pkg.UNet3D(precision="bf16", deterministic=True, dropout=0.0, **KW104).to(DEV)
        model.load_state_dict(sd)
        model.train()
        xd = x.to(DEV).requires_grad_(flagged)
        pkg.DiceLoss(sigmoid=True)(model(xd), t.to(DEV)).backward()
        torch.cuda.synchronize()
        runs[flagged] = [p.grad.clone() for p in model.ordered_parameters()]
        if flagged:
            assert xd.grad is not None and torch.isfinite(xd.grad).all()
    for a, b in zip(runs[False], runs[True]):
        assert torch.equal(a, b)


def test_graphed_train_step_runs_at_104_outputs(pkg):
    model = pkg.UNet3D(precision="bf16", dropout=0.0, **KW104).to(DEV)
    model.train()
    crit = pkg.DiceLoss(sigmoid=True)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    step = pkg.train.GraphedTrainStep(model, crit, opt, (2, 2, 16, 16, 16), (2, 104, 16, 16, 16))
    losses = []
    for i in range(3):
        x, t = _batch(20 + i, shape=(2, 2, 16, 16, 16))
        losses.append(float(step(x.pin_memory(), t.pin_memory()).item()))
    assert all(0.0 < v < 1.0 for v in losses)


def test_sliding_window_inference_at_104_outputs(pkg):
    kw = dict(n_features=2, n_outputs=104, base_width=8)
    cfg = UNetConfig(**kw)
    sd = make_state_dict(cfg, seed=4)
    model = pkg.UNet3D(precision="split", **kw).to(DEV)
    model.load_state_dict(sd)
    model.eval()
    x = torch.randn(1, 2, 24, 20, 28, generator=torch.Generator().manual_seed(1))
    inf = pkg.predict.SlidingWindowInferer(roi_size=(16, 16, 16), sw_batch_size=4, overlap=0.25, mode="gaussian")
    with torch.no_grad():
        got = inf(x.to(DEV), model).cpu()
        ref = sliding_window_inference(x.double(), (16, 16, 16), lambda tiles: unet3d_forward({k: v.double() for k, v in sd.items()}, tiles, cfg),
                                       overlap=0.25, mode="gaussian")
    assert got.shape == (1, 104, 24, 20, 28)
    assert _rel(got, ref) < 1e-3


# ------------------------------------------------------------------------------------------------ pre/post-processing, 104 channels
def test_one_hot_104_labels_bit_exact(pkg, gold):
    data = one_hot_input()
    got = pkg.prepost.compile_one_hot_encoding(data.to(DEV), n_labels=N_LABELS, return_4d=False).cpu().numpy()
    shp = tuple(int(v) for v in gold["one_hot104_shape"])
    ref = np.unpackbits(gold["one_hot104"])[: int(np.prod(shp))].reshape(shp)
    assert got.shape == shp and (got == ref).all()
    assert (got == one_hot_encode(data.numpy(), N_LABELS)).all()


@pytest.mark.parametrize("name", sorted(LABEL_MAP_CASES))
def test_label_map_104_channels_bit_exact(pkg, gold, name):
    p = label_map_prediction()
    got = pkg.prepost.convert_one_hot_to_label_map(p.to(DEV), labels=labels(), **LABEL_MAP_CASES[name]).cpu().numpy()
    assert (got == gold[name]).all()
    assert (got == label_map_from_one_hot(p.numpy(), labels(), **LABEL_MAP_CASES[name])).all()


def test_label_map_104_channels_fused_softmax(pkg):
    logits = torch.randn(N_LABELS, 6, 7, 8, generator=torch.Generator().manual_seed(9)) * 3
    got = pkg.prepost.convert_one_hot_to_label_map(logits.to(DEV), labels(), activation="softmax", threshold=0.05).cpu().numpy()
    ref = label_map_from_one_hot(torch.softmax(logits, dim=0).numpy(), labels(), threshold=0.05)
    assert (got != ref).mean() < 1e-3
