"""MONAI UNet at the sizes README times it: channels (16, 32, 64, 128, 256), num_res_units 2, PReLU, instance norm, trained with
DiceCELoss(softmax=True, to_onehot_y=True) -- spleen, 1 -> 2 channels at 4 x 96^3, and BraTS, 4 -> 3 channels at 2 x 128^3 with
the input gradient -- against the oracle (oracle/unet_oracle.py + tests/dice_ce_oracle.py) in fp64 on the CPU.  At these sizes
the plans run what the small networks of test_gpu_monai_unet.py never reach: a 384-channel concat into the 384 -> 64 transposed
conv (6 K chunks), 256 -> 256 convs and data gradients (4), the 128 -> 256 1x1x1 residual, BN 128 per-tap tiles on 6^3 and 8^3
outputs, stride-2 convs on the packed 1- and 4-channel input with their parity-class data gradients, the two-CTA (BN 64, KC 64)
halo kernel (BraTS bf16, 64 -> 64 at 16^3), weight gradients split over every SM at 48^3-64^3 and over 4-16 splits at the
bottom, PReLU slope gradients over up to 8 M voxel-channels, instance norm over 216 voxels per channel, and a 5-level
forward-only plan that recycles its buffers.  The routes of every convolution and weight gradient are asserted against
monai_unet_cases.ROUTES / WGRAD_ROUTES on a 132-SM H100.

Bounds: split precision those of test_gpu_monai_unet.py (its check_split_grads: logits rel-L2 <= 1e-3, gradient norms within
3 % and cosine > 0.999, the noise-floor rule for the PReLU slopes, the absolute bound for the conv biases in front of an instance
norm, the input gradient rel-L2 <= 5e-2) and the loss within 1e-3 relative; bf16 logits rel-L2 <= 1.25x the rel-L2 of torch's
bf16 autocast on the oracle's graph, weights and input (as test_gpu_c5_size.py), the loss within 1e-3 relative, every gradient
finite; the forward-only plan's logits against the training plan's forward within rel-L2 1e-6, in a smaller workspace;
deterministic bf16 gradients bit-identical over two steps at spleen size.

Measured on an H100 80GB HBM3 at 700 W, the oracle on 8 CPU threads (its forward, loss and backward; then two perturbed passes
for the slopes' noise floor):
  spleen  oracle 14.6 s (37.6 s with the floor); split logits rel-L2 1.8e-5, loss 4.3e-8 relative, worst gradient-norm
          deviation 5.6e-4; bf16 logits 9.6e-3 against autocast's 1.15e-2 (ratio 0.83), loss 1.0e-5 relative; peak device memory
          2.4 GiB (split) and 1.3 GiB (bf16, with autocast); forward-only plan bit-identical in a 0.52 GiB workspace (1.22 GiB)
  BraTS   oracle 16.1 s (39.4 s); split 1.4e-5, loss 8.7e-8, worst 2.6e-4, input gradient 7.1e-3; bf16 7.3e-3 against 8.9e-3
          (0.82), loss 3.5e-5; peak 3.1 and 1.75 GiB; forward-only plan bit-identical in 0.62 GiB (1.43 GiB)
Each GPU test takes 0.3-1.1 s after its workload's oracle; the module about 93 s.
"""
import time

import pytest
import torch

import monai_unet_cases as U
from dice_ce_oracle import dice_ce_loss
from oracle.unet_oracle import MonaiUNetConfig, make_unet_state_dict, unet_forward
from test_gpu_monai_unet import BOUNDS, _kw, _reference, _slope_noise_floor, check_split_grads, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"
CHANNELS = (16, 32, 64, 128, 256)
# (batch, in, out, extents) of tools/monai_unet_bench.py; BraTS also computes the input gradient (monai_unet_cases: brats)
WORKLOADS = {"spleen": (4, 1, 2, (96, 96, 96)), "brats": (2, 4, 3, (128, 128, 128))}
INPUT_GRAD = {"spleen": False, "brats": True}
LOSS_REL = 1e-3


def _cfg(name):
    n, cin, cout, dims = WORKLOADS[name]
    return MonaiUNetConfig(cin, cout, CHANNELS, 2, "prelu")


def _inputs(name, seed):
    n, cin, cout, dims = WORKLOADS[name]
    g = torch.Generator().manual_seed(100 + seed)
    x = torch.randn((n, cin) + dims, generator=g, dtype=torch.float64)
    t = torch.randint(0, cout, (n, 1) + dims, generator=g).to(torch.uint8)
    return make_unet_state_dict(_cfg(name), seed=seed), x, t


def _loss(t):
    return lambda out: dice_ce_loss(out, t, softmax=True, to_onehot_y=True)


@pytest.fixture(scope="module", params=list(WORKLOADS))
def oracle(request):
    """fp64 CPU forward + DiceCELoss + backward of the oracle: logits, loss, every parameter gradient, the input gradient, and
    the PReLU slopes' noise floor"""
    name = request.param
    cfg = _cfg(name)
    sd, x, t = _inputs(name, seed=3 if name == "spleen" else 4)
    t0 = time.perf_counter()
    loss = _loss(t)
    out, grads, dx = _reference(cfg, sd, x, None, loss)
    with torch.no_grad():
        value = float(loss(out))
    seconds = time.perf_counter() - t0
    floor = _slope_noise_floor(cfg, sd, x, None, grads, loss=loss)
    print("\nMONAI UNet %s CPU oracle (fp64, %d threads): %.1f s, with the slopes' noise floor %.1f s"
          % (name, torch.get_num_threads(), seconds, time.perf_counter() - t0))
    return dict(name=name, cfg=cfg, sd=sd, x=x, t=t, logits=out, loss=value, grads=grads, dx=dx, floor=floor)


def _model(pkg, o, precision, deterministic=None):
    m = pkg.UNet(precision=precision, deterministic=deterministic, **_kw(o["cfg"])).to(DEV)
    m.load_state_dict({k: v.float() for k, v in o["sd"].items()}, strict=True)
    return m.train()


def _step(pkg, m, x, t, input_grad):
    """one forward, DiceCELoss and backward: (logits, loss, input gradient or None)"""
    xg = x.float().to(DEV).requires_grad_(input_grad)
    out = m(xg)
    loss = pkg.DiceCELoss(softmax=True, to_onehot_y=True)(out, t.to(DEV))
    loss.backward()
    torch.cuda.synchronize()
    return out.detach(), float(loss), xg.grad if input_grad else None


@pytest.mark.parametrize("precision", ["bf16", "split"])
@pytest.mark.parametrize("name", list(WORKLOADS))
def test_routes(pkg, name, precision):
    L = pkg.lib
    L.load_library()
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the route tables are for a 132-SM H100")
    config = next(c for c in U.CONFIGS if c.name == name)
    assert config.input_grad == INPUT_GRAD[name]
    assert U.route_table(L, config, precision == "split") == U.ROUTES[name][precision]
    assert U.wgrad_route_table(L, config, precision == "split") == U.WGRAD_ROUTES[name][precision]


def test_split_precision_matches_oracle(pkg, oracle):
    name = oracle["name"]
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    m = _model(pkg, oracle, "split")
    out, loss, dx = _step(pkg, m, oracle["x"], oracle["t"], INPUT_GRAD[name])
    rel = rel_l2(out, oracle["logits"])
    dloss = abs(loss - oracle["loss"]) / abs(oracle["loss"])
    worst = check_split_grads(m, oracle["grads"], oracle["floor"])
    rel_dx = rel_l2(dx, oracle["dx"]) if dx is not None else float("nan")
    print("\n%s split: logits rel-L2 %.3e, loss rel %.3e, worst gradient-norm deviation %.3e, input gradient rel-L2 %.3e "
          "(%.1f s, peak %.2f GiB)" % (name, rel, dloss, worst, rel_dx, time.perf_counter() - t0,
                                       torch.cuda.max_memory_allocated() / 2 ** 30))
    assert rel <= BOUNDS["logits"]
    assert dloss <= LOSS_REL
    if dx is not None:
        assert rel_dx <= BOUNDS["dx"]


def test_bf16_matches_fp64_at_autocast_class(pkg, oracle):
    name = oracle["name"]
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            p = {k: v.float().to(DEV) for k, v in oracle["sd"].items()}
            autocast = unet_forward(oracle["x"].float().to(DEV), p, oracle["cfg"]).double().cpu()
            del p
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    torch.cuda.empty_cache()
    m = _model(pkg, oracle, "bf16")
    out, loss, dx = _step(pkg, m, oracle["x"], oracle["t"], INPUT_GRAD[name])
    ours, theirs = rel_l2(out, oracle["logits"]), rel_l2(autocast, oracle["logits"])
    dloss = abs(loss - oracle["loss"]) / abs(oracle["loss"])
    print("\n%s bf16: logits rel-L2 %.3e, torch bf16 autocast %.3e, ratio %.3f, loss rel %.3e (%.1f s, peak %.2f GiB)"
          % (name, ours, theirs, ours / theirs, dloss, time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30))
    assert ours <= 1.25 * theirs
    assert dloss <= LOSS_REL
    for k, p in m.named_parameters():
        assert bool(torch.isfinite(p.grad).all()), k
    if dx is not None:
        assert bool(torch.isfinite(dx).all())


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_forward_only_plan_matches_training_plan_forward(pkg, name):
    """bf16: the forward-only plan recycles released buffers over five levels; the training plan keeps every activation"""
    sd, x, _ = _inputs(name, seed=5)
    m = _model(pkg, dict(sd=sd, cfg=_cfg(name)), "bf16")
    xd = x.float().to(DEV)
    train = m(xd)
    assert train.requires_grad
    train = train.detach()
    with torch.no_grad():
        fwd_only = m(xd)
    torch.cuda.synchronize()
    plans = {k[-1]: p for k, p in m._plans.items()}
    assert set(plans) == {True, False}
    ws_infer, ws_train = plans[True].ws_bytes, plans[False].ws_bytes
    rel = rel_l2(fwd_only, train)
    print("\n%s forward-only vs training plan: rel-L2 %.3e, workspaces %.2f / %.2f GiB"
          % (name, rel, ws_infer / 2 ** 30, ws_train / 2 ** 30))
    assert rel <= 1e-6
    assert ws_infer < ws_train


def test_spleen_deterministic_gradients_bit_identical(pkg):
    sd, x, t = _inputs("spleen", seed=6)
    m = _model(pkg, dict(sd=sd, cfg=_cfg("spleen")), "bf16", deterministic=True)
    grads = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        _step(pkg, m, x, t, False)
        grads.append({k: p.grad.clone() for k, p in m.named_parameters()})
    for k in grads[0]:
        assert torch.equal(grads[0][k], grads[1][k]), k
