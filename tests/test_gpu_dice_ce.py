"""DiceCELoss on the GPU: the fused kernels against the hand-derived values and fp64 autograd of the torch-op restatement
(tests/dice_ce_oracle.py) for every target form, activation and Dice flag at 1..128 classes, out-of-range labels, run-to-run
bit equality, a UNet3D training step on a label map, and CUDA-graph steps on label maps."""
import pytest
import torch

from oracle import UNetConfig, make_state_dict, unet3d_forward
from oracle.dynunet_oracle import make_dynunet_state_dict
from dice_ce_oracle import dice_ce_loss
from test_dice_ce_host import X, T

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


def _cos(a, b):
    a, b = a.double().cpu().ravel(), b.double().cpu().ravel()
    return float((a * b).sum() / (a.norm() * b.norm() + 1e-300))


def _run(pkg, x, t, **kw):
    """fused loss and dlogits (grad_out = 1)"""
    xx = x.detach().to(DEV).float().requires_grad_(True)
    loss = pkg.DiceCELoss(**kw)(xx, t.to(DEV))
    loss.backward()
    return float(loss.detach()), xx.grad.detach().double().cpu()


def _oracle(x, t, **kw):
    okw = {k: v for k, v in kw.items() if k != "to_onehot_y"}
    xx = x.detach().double().to(DEV).requires_grad_(True)
    loss = dice_ce_loss(xx, t.to(DEV), **okw)
    loss.backward()
    return float(loss.detach()), xx.grad.detach().cpu()


@pytest.mark.parametrize("kw, expected", [
    (dict(to_onehot_y=True), 0.313262),
    (dict(to_onehot_y=True, softmax=True), 0.599181),
    (dict(to_onehot_y=True, softmax=True, lambda_ce=2.0), 0.912443),
    (dict(to_onehot_y=True, include_background=False), 0.313262),
])
def test_known_answers(pkg, kw, expected):
    v, _ = _run(pkg, X, T.to(torch.uint8), **kw)
    assert abs(v - expected) < 1e-6, v
    vo, _ = _oracle(X, T, **kw)
    assert abs(v - vo) < 1e-6


def _inputs(c, form, act, spatial, seed):
    g = torch.Generator().manual_seed(seed)
    shape = (2, c) + spatial
    # identity activation: probabilities as MONAI's own tests feed them (raw logits would make the Dice denominators arbitrary)
    identity = act is None or (act == "softmax" and c == 1)      # with one channel softmax is ignored
    x = torch.rand(shape, generator=g) if identity else 2.0 * torch.randn(shape, generator=g)
    lshape = (2, 1) + spatial
    if c == 1:
        b = torch.rand(lshape, generator=g) > 0.5
        t = {"label_u8": b.to(torch.uint8), "label_i64": b.long(), "onehot_u8": b.to(torch.uint8),
             "soft_f32": torch.rand(lshape, generator=g)}[form]
        return x, t, False
    lab = torch.randint(0, c, lshape, generator=g)
    if form == "label_u8":
        return x, lab.to(torch.uint8), True
    if form == "label_i64":
        return x, lab, True
    if form == "onehot_u8":
        return x, torch.nn.functional.one_hot(lab[:, 0], c).movedim(-1, 1).to(torch.uint8), False
    return x, torch.softmax(torch.randn(shape, generator=g), dim=1), False


VARIANTS = [dict(), dict(include_background=False), dict(batch=True), dict(squared_pred=True), dict(jaccard=True),
            dict(reduction="sum"), dict(lambda_dice=0.3, lambda_ce=1.7), dict(lambda_ce=0.0),
            dict(include_background=False, batch=True, squared_pred=True, jaccard=True)]


@pytest.mark.parametrize("spatial", [(3, 5, 7), (24, 32, 40)])
@pytest.mark.parametrize("act", [None, "sigmoid", "softmax"])
@pytest.mark.parametrize("form", ["label_u8", "label_i64", "onehot_u8", "soft_f32"])
@pytest.mark.parametrize("c", [1, 2, 3, 16, 104, 128])
def test_kernels_match_fp64_oracle_autograd(pkg, c, form, act, spatial):
    x, t, onehot_y = _inputs(c, form, act, spatial, seed=c * 131 + len(form) * 7 + spatial[0])
    for var in VARIANTS:
        kw = dict(var, to_onehot_y=onehot_y, sigmoid=act == "sigmoid", softmax=act == "softmax")
        v, g = _run(pkg, x, t, **kw)
        vo, go = _oracle(x, t, **kw)
        assert abs(v - vo) <= 1e-5 * abs(vo), (kw, v, vo)
        assert _rel(g, go) <= 1e-4, (kw, _rel(g, go))


@pytest.mark.parametrize("c", [2, 16, 104])
def test_label_map_and_one_hot_agree(pkg, c):
    x, lab, _ = _inputs(c, "label_u8", "softmax", (17, 19, 23), seed=3)
    oh = torch.nn.functional.one_hot(lab[:, 0].long(), c).movedim(-1, 1).to(torch.uint8)
    for var in VARIANTS[:6]:
        v1, g1 = _run(pkg, x, lab, softmax=True, to_onehot_y=True, **var)
        v2, g2 = _run(pkg, x, oh, softmax=True, **var)
        assert abs(v1 - v2) <= 1e-6 * abs(v2)
        assert _rel(g1, g2) <= 1e-6


@pytest.mark.parametrize("dtype, bad", [(torch.uint8, 200), (torch.int64, 7), (torch.int64, -1)])
def test_out_of_range_labels_are_all_zero_rows(pkg, dtype, bad):
    g = torch.Generator().manual_seed(11)
    x = 2.0 * torch.randn(2, 3, 6, 7, 9, generator=g)
    lab = torch.randint(0, 3, (2, 1, 6, 7, 9), generator=g)
    lab[torch.rand(lab.shape, generator=g) < 0.2] = bad
    lab = lab.to(dtype)
    for kw in (dict(softmax=True), dict(sigmoid=True, batch=True), dict(softmax=True, include_background=False)):
        v, gr = _run(pkg, x, lab, to_onehot_y=True, **kw)
        vo, go = _oracle(x, lab, **kw)
        assert abs(v - vo) <= 1e-5 * abs(vo)
        assert _rel(gr, go) <= 1e-4


def test_bit_identical_run_to_run_at_104_classes(pkg):
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 104, 64, 64, 64, generator=g).to(DEV)
    lab = torch.randint(0, 104, (2, 1, 64, 64, 64), generator=g).to(torch.uint8).to(DEV)
    crit = pkg.DiceCELoss(softmax=True, to_onehot_y=True)
    runs = []
    for _ in range(2):
        xx = x.clone().requires_grad_(True)
        loss = crit(xx, lab)
        loss.backward()
        torch.cuda.synchronize()
        runs.append((loss.detach().clone(), xx.grad.clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_unet3d_16_class_step_on_a_label_map(pkg):
    kw = dict(n_features=4, n_outputs=16, base_width=8)
    cfg = UNetConfig(**kw)
    sd = make_state_dict(cfg, seed=3)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(1, 4, 32, 32, 32, generator=g)
    lab = torch.randint(0, 16, (1, 1, 32, 32, 32), generator=g).to(torch.uint8)
    sd64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    ref = unet3d_forward(sd64, x.double(), cfg, dropout_mask=torch.ones(1, 8))
    lref = dice_ce_loss(ref, lab, softmax=True)
    lref.backward()
    model = pkg.UNet3D(precision="split", **kw).to(DEV)
    model.load_state_dict(sd, strict=True)
    model.train()
    model.set_dropout_scale(torch.ones(1, 8))
    out = model(x.to(DEV))
    loss = pkg.DiceCELoss(softmax=True, to_onehot_y=True)(out, lab.to(DEV))
    loss.backward()
    assert _rel(out.detach(), ref.detach()) < 1e-3
    assert abs(float(loss.detach()) / float(lref.detach()) - 1) < 1e-3
    for k, p in model.named_parameters():
        r = sd64[k].grad
        assert abs(float(p.grad.double().norm()) / float(r.norm()) - 1) < 3e-2, k
        assert _cos(p.grad, r) > 0.999, k


def _dynunet(pkg):
    kw = dict(spatial_dims=3, in_channels=2, out_channels=5, kernel_size=[[3, 3, 3]] * 3, strides=[[1, 1, 1]] + [[2, 2, 2]] * 2,
              upsample_kernel_size=[[2, 2, 2]] * 2, filters=[16, 24, 32])
    model = pkg.DynUNet(precision="split", **kw).to(DEV)
    model.load_state_dict(make_dynunet_state_dict(2, 5, kw["filters"], seed=4), strict=True)
    model.train()
    return model


def _label_batch(seed, n=2, c_in=2, c_out=5, s=16):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, c_in, s, s, s, generator=g), torch.randint(0, c_out, (n, 1, s, s, s), generator=g).to(torch.uint8)


def test_graphed_step_replays_the_eager_label_map_loss(pkg):
    model = _dynunet(pkg)
    crit = pkg.DiceCELoss(softmax=True, to_onehot_y=True)
    x, lab = _label_batch(1)
    eager = crit(model(x.to(DEV)), lab.to(DEV))
    eager.backward()
    eager_v = float(eager.detach())
    del eager
    model.zero_grad(set_to_none=True)
    opt = torch.optim.SGD(model.parameters(), lr=0.0)
    step = pkg.train.GraphedTrainStep(model, crit, opt, tuple(x.shape), tuple(lab.shape), target_dtype=torch.uint8)
    for _ in range(2):
        v = float(step(x.pin_memory(), lab.pin_memory()).item())
        assert abs(v / eager_v - 1) < 1e-6, (v, eager_v)


def test_epoch_training_with_cuda_graph_on_label_maps(pkg):
    model = _dynunet(pkg)
    crit = pkg.DiceCELoss(softmax=True, to_onehot_y=True)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    loader = []
    for i in range(3):
        x, lab = _label_batch(30 + i)
        loader.append({"image": x, "label": lab})
    seen = []

    class Recording:
        def __init__(self, inner):
            self.inner = inner

        def __call__(self, out, t):
            seen.append((tuple(t.shape), t.dtype))
            return self.inner(out, t)
    avg = pkg.train.epoch_training(loader, model, Recording(crit), opt, epoch=0, n_gpus=1, print_frequency=0, use_cuda_graph=True)
    assert torch.isfinite(torch.tensor(avg)) and avg > 0.0
    assert all(s == ((2, 1, 16, 16, 16), torch.uint8) for s in seen)
    assert len(model._graphed_steps) == 1
