"""DynUNet at the size its example config trains it (examples/brats2020/brats2020_config.json, plan_launches.BRATS_DYNUNET: six
levels, filters 64/96/128/192/256/384, 4 -> 3 channels), batch 2 of 4 x 128^3 with DiceLoss(sigmoid=True), against the oracle
(oracle/dynunet_oracle.py).  At this size the plan runs what the small networks of test_gpu_dynunet.py never reach: a 4^3
bottleneck whose 256 -> 384 stride-2 and 384 -> 384 convs produce 128 voxels per launch (less than one 256-voxel tile) and whose
instance norms average 64 voxels per channel; the 384 -> 256 transposed conv (6 K chunks) with its data and weight gradients;
the concat-source convs 512 -> 256 .. 128 -> 64, the last at 128^3; the 64 -> 64 convs and data gradients at 128^3 on the
two-CTA (BN 64, KC 64) halo kernel in bf16; parity-class data gradients onto 64^3 and 128^3; weight gradients over 4.2 M voxels
and over 128 at the bottom; the biased head's bias gradient over 4.2 M voxels; and the input gradient.  The routes of every
convolution and weight gradient are asserted against dynunet_cases.BRATS_ROUTES / BRATS_WGRAD_ROUTES on a 132-SM H100.

Oracle: dynunet_forward in fp64 on the GPU through cuDNN, one sample at a time, pinned to the CPU oracle by
test_gpu_fp64_graph_is_the_cpu_oracle below.  Instance norm and the Dice loss (batch=False, mean over samples and channels) are
per sample, so the batch loss is the mean of the per-sample losses and every gradient the mean of theirs.  One step is about
8.1e12 multiply-adds, some 10 minutes of torch's CPU convolutions; the same graph runs again in fp32 under torch's bf16 autocast.
Its results go to the host and its tensors are freed before any plan runs.  A plan that drops the last K chunk of the 512-channel
concat source (upsamples.0.conv_block.conv1) fails the split test: logits rel-L2 8.1e-2, input gradient cosine 0.72.

Bounds: split precision those of test_gpu_dynunet.py (logits rel-L2 <= 1e-3, |dDice| <= 1e-3 |Dice|, every gradient norm within
3 % and cosine > 0.999, 0.995 for tensors of at most 64 elements) and, for the input gradient, those of test_gpu_input_grad.py
(norm within 3 %, cosine > 0.999); bf16 those of test_gpu_bf16_vs_autocast.py against torch's bf16 autocast on the same graph,
weights and input (logits <= 2e-2 and <= 1.25x autocast's rel-L2, loss within 1e-3 relative, whole gradient <= 1.25x autocast,
median per-tensor ratio <= 1.25, every tensor <= 2x autocast + 5e-3, every gradient norm within 8 %); the forward-only plan
against the training plan's forward, and each sample of the batch-2 forward against its batch-1 forward, within rel-L2 1e-6;
deterministic bf16 gradients bit-identical over two steps, and a captured CUDA-graph step replaying the eager loss and gradients.

Measured on an H100 80GB HBM3 at 700 W:
  oracle   fp64 7.1 s at a peak of 18.7 GiB of device memory; bf16 autocast 1.3 s, 4.8 GiB
  split    logits rel-L2 3.8e-5, loss 5.1e-8 relative, worst gradient-norm deviation 6.6e-3 (downsamples.0.norm1.bias), lowest
           cosine 0.99969; input gradient rel-L2 1.7e-2, norm 7.1e-5 off, cosine 0.99985; peak 26.8 GiB
  bf16     logits rel-L2 1.63e-2 against autocast's 1.66e-2 (ratio 0.98), loss 4.8e-6 relative; whole gradient 3.68e-2 against
           3.73e-2 (0.99), median per-tensor ratio 0.99, worst gradient-norm deviation 5.9e-2; peak 13.5 GiB
  the forward-only plan and the batch-1 forwards are bit-identical to the training plan's and the batch-2 forward, in a 3.79 GiB
  workspace against 13.12 GiB; the graphed step replays the eager loss and gradients bit for bit.
Each GPU test takes under a second after the oracle; the module about 36 s.
"""
import time

import pytest
import torch

import dynunet_cases as D
import plan_launches as P
from oracle import dice_loss
from oracle.dynunet_oracle import dynunet_forward, make_dynunet_state_dict
from segresnet_cases import RELU_BOUNDS as BOUNDS
from test_gpu_bf16_vs_autocast import check_autocast_class
from test_gpu_monai_unet import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"
KW = P.BRATS_DYNUNET
LEVELS = len(KW["filters"])
SHAPE = (D.BRATS.n, KW["in_channels"]) + D.BRATS.dims
SEED = 8


def _inputs(kw, shape, seed):
    """fp32 state dict, fp32 input and uint8 Dice target"""
    sd = make_dynunet_state_dict(kw["in_channels"], kw["out_channels"], kw["filters"], seed=seed)
    g = torch.Generator().manual_seed(100 + seed)
    x = torch.randn(shape, generator=g)
    t = (torch.rand((shape[0], kw["out_channels"]) + tuple(shape[2:]), generator=g) > 0.7).to(torch.uint8)
    return sd, x, t


def _oracle_on_gpu(sd, x, t, levels, dtype, autocast=False):
    """forward, sigmoid Dice and backward of the oracle graph on the device, one sample at a time, each loss divided by the batch:
    (logits, loss, {key: gradient}, input gradient), on the host in fp64"""
    n = x.shape[0]
    p = {k: v.to(DEV, dtype).requires_grad_(True) for k, v in sd.items()}
    outs, dxs, loss = [], [], 0.0
    for i in range(n):
        xi = x[i:i + 1].to(DEV, dtype).requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            out = dynunet_forward(p, xi, levels)
        li = dice_loss(out.float() if autocast else out, t[i:i + 1].to(DEV)) / n
        li.backward()
        loss += float(li.detach())
        outs.append(out.detach().double().cpu())
        dxs.append(xi.grad.double().cpu())
        del out, li, xi
    grads = {k: v.grad.double().cpu() for k, v in p.items()}
    del p
    return torch.cat(outs), loss, grads, torch.cat(dxs)


def test_gpu_fp64_graph_is_the_cpu_oracle():
    """the ground truth below (the oracle graph on the device in fp64, sample by sample) against the CPU oracle in fp64 on the
    whole batch: 4 levels, so the transposed convs and the concats are in it"""
    kw = dict(in_channels=4, out_channels=3, filters=[8, 16, 24, 32])
    sd, x, t = _inputs(kw, (2, 4, 16, 16, 16), seed=1)
    out_g, loss_g, grads_g, dx_g = _oracle_on_gpu(sd, x, t, 4, torch.float64)
    sdc = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    xc = x.double().requires_grad_(True)
    out_c = dynunet_forward(sdc, xc, 4)
    loss_c = dice_loss(out_c, t)
    loss_c.backward()
    assert rel_l2(out_g, out_c.detach()) < 1e-10
    assert abs(loss_g - float(loss_c.detach())) < 1e-12
    for k in sdc:
        assert rel_l2(grads_g[k], sdc[k].grad) < 1e-8, k
    assert rel_l2(dx_g, xc.grad) < 1e-8


@pytest.fixture(scope="module")
def oracle():
    """the seeded weights, input and target; the fp64 logits, loss, gradients and input gradient; and the same of torch's bf16
    autocast (fp32 parameters, TF32 off)"""
    sd, x, t = _inputs(KW, SHAPE, SEED)
    res = dict(sd=sd, x=x, t=t)
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for name, dtype, autocast in (("ref", torch.float64, False), ("autocast", torch.float32, True)):
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            res[name] = _oracle_on_gpu(sd, x, t, LEVELS, dtype, autocast)
            torch.cuda.synchronize()
            print("\nDynUNet BraTS oracle on the device (%s, 2 samples of 4 x 128^3): %.1f s, peak %.1f GiB"
                  % (name, time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    torch.cuda.empty_cache()
    return res


def _model(pkg, sd, precision, deterministic=None):
    m = pkg.DynUNet(precision=precision, deterministic=deterministic, **KW).to(DEV)
    m.load_state_dict(sd, strict=True)
    return m.train()


def _step(pkg, m, x, t, input_grad=False):
    """one forward, sigmoid Dice and backward: (logits, loss, {key: gradient}, input gradient or None), on the host in fp64"""
    xd = x.to(DEV).requires_grad_(input_grad)
    out = m(xd)
    loss = pkg.DiceLoss(sigmoid=True)(out, t.to(DEV))
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.double().cpu() for k, p in m.named_parameters()}
    return out.detach().double().cpu(), float(loss), grads, xd.grad.double().cpu() if input_grad else None


def _infer(m, x):
    with torch.no_grad():
        out = m(x.to(DEV))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("precision", ["bf16", "split"])
def test_routes(pkg, precision):
    L = pkg.lib
    L.load_library()
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the route tables are for a 132-SM H100")
    assert D.route_table(L, precision == "split") == D.BRATS_ROUTES[precision]
    assert D.wgrad_route_table(L, precision == "split") == D.BRATS_WGRAD_ROUTES[precision]


def test_split_precision_matches_fp64(pkg, oracle):
    """every parameter gradient and the input gradient (key "x") held to a norm within 3 % and a cosine above 0.999 (0.995 for at
    most 64 elements)"""
    ref_out, ref_loss, ref_g, ref_dx = oracle["ref"]
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    m = _model(pkg, oracle["sd"], "split")
    out, loss, grads, dx = _step(pkg, m, oracle["x"], oracle["t"], input_grad=True)
    seconds, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30
    del m
    torch.cuda.empty_cache()
    rel, dloss = rel_l2(out, ref_out), abs(loss - ref_loss) / abs(ref_loss)
    assert set(grads) == set(ref_g)
    grads["x"], ref_g = dx, dict(ref_g, x=ref_dx)
    dev = {k: abs(float(g.norm() / ref_g[k].norm()) - 1.0) for k, g in grads.items()}
    cos = {k: float((g * ref_g[k]).sum() / (g.norm() * ref_g[k].norm() + 1e-300)) for k, g in grads.items()}
    worst = max((v, k) for k, v in dev.items() if k != "x")
    print("\nsplit: logits rel-L2 %.3e, loss rel %.3e, worst gradient-norm deviation %.3e (%s), lowest cosine %.6f (%s), input "
          "gradient rel-L2 %.3e, norm deviation %.3e, cosine %.6f (%.1f s, peak %.2f GiB)"
          % (rel, dloss, worst[0], worst[1], *min((v, k) for k, v in cos.items()), rel_l2(dx, ref_dx), dev["x"], cos["x"],
             seconds, peak))
    assert rel <= BOUNDS["logits"]
    assert dloss <= BOUNDS["loss"]
    for k, g in grads.items():
        assert bool(torch.isfinite(g).all()), k
        assert dev[k] < BOUNDS["grad_norm"], (k, dev[k])
        assert cos[k] > (BOUNDS["cos_small"] if g.numel() <= 64 else BOUNDS["cos"]), (k, cos[k])


def test_bf16_matches_fp64_at_autocast_class(pkg, oracle):
    ref_out, ref_loss, ref_g, _ = oracle["ref"]
    ac_out, _, ac_g, _ = oracle["autocast"]
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    m = _model(pkg, oracle["sd"], "bf16")
    out, loss, grads, _ = _step(pkg, m, oracle["x"], oracle["t"])
    seconds, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30
    del m
    torch.cuda.empty_cache()
    ours, theirs = rel_l2(out, ref_out), rel_l2(ac_out, ref_out)
    dloss = abs(loss - ref_loss) / abs(ref_loss)
    assert all(bool(torch.isfinite(g).all()) for g in grads.values())
    whole, whole_ac, median, worst = check_autocast_class(grads, ac_g, ref_g)
    print("\nbf16: logits rel-L2 %.3e, torch bf16 autocast %.3e, ratio %.3f, loss rel %.3e; whole gradient rel-L2 %.3e against "
          "autocast's %.3e (ratio %.3f), median per-tensor ratio %.3f, worst gradient-norm deviation %.3e (%.1f s, peak %.2f GiB)"
          % (ours, theirs, ours / theirs, dloss, whole, whole_ac, whole / whole_ac, median, worst, seconds, peak))
    assert ours <= 2e-2
    assert ours <= 1.25 * theirs
    assert dloss <= 1e-3


def test_forward_only_plan_matches_training_plan_forward(pkg, oracle):
    """bf16, eval: the forward-only plan recycles released buffers over six levels; the training plan keeps every activation"""
    m = _model(pkg, oracle["sd"], "bf16").eval()
    fwd_only = _infer(m, oracle["x"])
    train = m(oracle["x"].to(DEV))
    assert train.requires_grad
    train = train.detach().cpu()
    plans = {k[-1]: p for k, p in m._plans.items()}
    assert set(plans) == {True, False}
    ws_infer, ws_train = plans[True].ws_bytes, plans[False].ws_bytes
    del m
    torch.cuda.empty_cache()
    rel = rel_l2(fwd_only, train)
    print("\nforward-only vs training plan: rel-L2 %.3e, workspaces %.2f / %.2f GiB" % (rel, ws_infer / 2 ** 30, ws_train / 2 ** 30))
    assert rel <= 1e-6
    assert ws_infer < ws_train


def test_batch_of_two_matches_batches_of_one(pkg, oracle):
    """bf16 forward: the config trains at batch 1, the benchmark at 2; each sample's launches see the same tiles and statistics
    partial sums at either batch size"""
    m = _model(pkg, oracle["sd"], "bf16").eval()
    out = _infer(m, oracle["x"])
    one = torch.cat([_infer(m, oracle["x"][i:i + 1]) for i in range(SHAPE[0])])
    assert sorted(k[0] for k in m._plans) == [1, SHAPE[0]]
    del m
    torch.cuda.empty_cache()
    rels = [rel_l2(out[i], one[i]) for i in range(SHAPE[0])]
    print("\nbatch 2 vs batch 1: rel-L2 %s" % ", ".join("%.3e" % r for r in rels))
    assert max(rels) <= 1e-6


def test_deterministic_bf16_step_and_graphed_step(pkg, oracle):
    """two eager steps of a deterministic bf16 plan give bit-identical gradients; train.GraphedTrainStep (SGD, lr 0) captures the
    step and its replays give the eager loss and gradients"""
    m = _model(pkg, oracle["sd"], "bf16", deterministic=True)
    x, t = oracle["x"].to(DEV), oracle["t"].to(DEV)
    crit = pkg.DiceLoss(sigmoid=True)
    runs = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        loss = crit(m(x), t)
        loss.backward()
        runs.append((float(loss), [p.grad.clone() for p in m.ordered_parameters()]))
        del loss                  # no autograd graph of an eager step may be alive when the step is captured
    for k, a, b in zip(m._keys, runs[0][1], runs[1][1]):
        assert torch.equal(a, b), k
    loss_e, g_eager = runs[1]
    step = pkg.train.GraphedTrainStep(m, crit, torch.optim.SGD(m.parameters(), lr=0.0), tuple(x.shape), tuple(t.shape))
    for _ in range(3):
        loss_g = step(x, t)
    torch.cuda.synchronize()
    num = sum(float((a.double() - p.grad.double()).pow(2).sum()) for a, p in zip(g_eager, m.ordered_parameters())) ** 0.5
    den = sum(float(a.double().pow(2).sum()) for a in g_eager) ** 0.5
    print("\ngraphed vs eager step: |dloss| %.3e, gradient rel-L2 %.3e" % (abs(float(loss_g) - loss_e), num / den))
    assert abs(float(loss_g) - loss_e) < 1e-5
    assert num / den < 1e-4
