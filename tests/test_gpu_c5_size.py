"""The C5 inference network at the size bench.py times it: 1 channel, 5 levels [1, 2, 2, 4, 4], base_width 48 (widths 48 to 768),
three 128^3 tiles per forward on the forward-only plan, 27 tiles per 256^3 volume.  Its 384- and 768-channel convolutions walk 6
and 12 K chunks, and the forward-only plan recycles its temporaries (plan.cu: release_buf); no smaller plan test reaches either.

Oracle: the oracle's functional graph (oracle/unet3d_oracle.py) in fp64 on the GPU through torch/cuDNN, tile by tile, pinned to
the CPU oracle by test_gpu_bf16_vs_autocast.py::test_gpu_fp64_graph_is_the_cpu_oracle.  Its tensors are freed before the plan
runs.  Bounds: split precision per-sample logits rel-L2 <= 1e-3 (the north-star bound); bf16, the precision bench.py runs, logits
rel-L2 <= 2e-2 and <= 1.25x the rel-L2 of torch's bf16 autocast on the same graph, weights and tiles; a sample of the batch-3
forward against the batch-1 forward of its tile, the forward-only plan against the training plan's forward, and the device
sliding-window inferer (batches of three) against the oracle's window-by-window inferer driving the same model (batches of one),
each rel-L2 <= 1e-6: a sample's launches see the same tiles and statistics partial sums at every batch size, so only the order
of the fp64 statistics atomics differs.  The convolution routes of the forward are asserted against c5_cases.C5_ROUTES on a
132-SM H100.

Measured on an H100 80GB HBM3 at 700 W: the oracle takes 5.7 s for the three tiles in fp64 and in autocast, at a peak of 7.2 GiB
of device memory; split precision 2.3e-5 per tile; bf16 7.4e-3 against autocast's 7.8e-3 (ratio 0.95); the forward-only plan
is bit-identical to the training plan's forward, in a 2.68 GiB workspace against 7.69 GiB; the batch-3 forward is bit-identical
to the batch-1 forwards; the whole volume 2.9e-8.  Each test takes 2-4 s after the 4-8 s oracle."""
import time

import pytest
import torch

import c5_cases as C
from oracle import UNetConfig, make_state_dict, sliding_window_inference, unet3d_forward
from oracle.unet3d_oracle import _scan_starts

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 5


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


class _Meta(torch.Tensor):
    """the ``meta['filename_or_obj']`` volumetric_predictions reads from its inputs"""
    meta = None


@pytest.fixture(scope="module")
def oracle():
    """the seeded weights and 256^3 volume, the inferer's first three tiles, and per tile the fp64 and bf16-autocast logits"""
    cfg = UNetConfig(**C.C5)
    sd = make_state_dict(cfg, seed=SEED)
    vol = torch.randn((1, C.C5["n_features"]) + C.C5_VOLUME, generator=torch.Generator().manual_seed(100 + SEED))
    starts = [_scan_starts(s, r, C.C5_OVERLAP) for s, r in zip(C.C5_VOLUME, C.C5_ROI)]
    windows = [(d, h, w) for d in starts[0] for h in starts[1] for w in starts[2]][:C.C5_BATCH]
    rd, rh, rw = C.C5_ROI
    tiles = torch.cat([vol[:, :, d:d + rd, h:h + rh, w:w + rw] for d, h, w in windows]).contiguous()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    ref, ac = [], []
    try:
        with torch.no_grad():
            for dtype, autocast, dst in ((torch.float64, False, ref), (torch.float32, True, ac)):
                p = {k: v.to(DEV, dtype) for k, v in sd.items()}
                for i in range(C.C5_BATCH):
                    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                        dst.append(unet3d_forward(p, tiles[i:i + 1].to(DEV, dtype), cfg).double().cpu())
                del p
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    torch.cuda.empty_cache()
    print("\nC5 oracle (fp64 and bf16 autocast, 3 tiles of 128^3): %.1f s, peak %.1f GiB" % (time.perf_counter() - t0, peak))
    return dict(sd=sd, vol=vol, tiles=tiles, ref=torch.cat(ref), autocast=torch.cat(ac))


def _model(pkg, o, precision):
    m = pkg.UNet3D(precision=precision, **C.C5).to(DEV)
    m.load_state_dict(o["sd"], strict=True)
    m.eval()
    return m


def _infer(m, x):
    with torch.no_grad():
        out = m(x.to(DEV))
    torch.cuda.synchronize()
    return out.cpu()


def _inference_plans(m):
    """{batch: plan} of the forward-only plans the model has built"""
    return {k[0]: p for k, p in m._plans.items() if p.inference_only}


def test_c5_routes(pkg):
    L = pkg.lib
    L.load_library()
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the route table is for a 132-SM H100")
    for precision in ("bf16", "split"):
        assert C.route_table(L, precision == "split") == C.C5_ROUTES[precision]


def test_c5_split_precision_matches_fp64(pkg, oracle):
    t0 = time.perf_counter()
    m = _model(pkg, oracle, "split")
    out = _infer(m, oracle["tiles"])
    assert list(_inference_plans(m)) == [C.C5_BATCH]
    rels = [_rel(out[i], oracle["ref"][i]) for i in range(C.C5_BATCH)]
    print("\nC5 split: per-tile logits rel-L2 %s (%.1f s)" % (", ".join("%.3e" % r for r in rels), time.perf_counter() - t0))
    assert max(rels) <= 1e-3


def test_c5_bf16_matches_fp64_at_autocast_class(pkg, oracle):
    t0 = time.perf_counter()
    m = _model(pkg, oracle, "bf16")
    out = _infer(m, oracle["tiles"])
    ours, theirs = _rel(out, oracle["ref"]), _rel(oracle["autocast"], oracle["ref"])
    print("\nC5 bf16: logits rel-L2 %.3e, torch bf16 autocast %.3e, ratio %.3f (%.1f s)"
          % (ours, theirs, ours / theirs, time.perf_counter() - t0))
    assert ours <= 2e-2
    assert ours <= 1.25 * theirs


def test_c5_batch_of_three_matches_batch_of_one(pkg, oracle):
    """bf16: the batch-3 forward against the batch-1 forward of each tile.  The up-sampling's per-sample grid, which sets the
    voxels each fp32 partial sum of the concat buffers' statistics covers, is the same at every batch size (with a per-batch
    block budget tiles 0 and 2 moved by 3.7e-4 and 2.9e-4 through flipped bf16 roundings downstream)"""
    t0 = time.perf_counter()
    m = _model(pkg, oracle, "bf16")
    out = _infer(m, oracle["tiles"])
    one = torch.cat([_infer(m, oracle["tiles"][i:i + 1]) for i in range(C.C5_BATCH)])
    assert sorted(_inference_plans(m)) == [1, C.C5_BATCH]
    rels = [_rel(out[i], one[i]) for i in range(C.C5_BATCH)]
    print("\nC5 batch 3 vs batch 1: rel-L2 %s (%.1f s)" % (", ".join("%.3e" % r for r in rels), time.perf_counter() - t0))
    assert max(rels) <= 1e-6


def test_c5_forward_only_plan_matches_training_plan_forward(pkg, oracle):
    """the forward-only plan recycles released buffers; the training plan keeps every activation for the backward"""
    t0 = time.perf_counter()
    m = _model(pkg, oracle, "bf16")
    x = oracle["tiles"][:1].to(DEV)
    fwd_only = _infer(m, x)
    train = m(x)                       # eval, grad enabled: the training plan (its activations are kept for a backward)
    assert train.requires_grad
    train = train.detach().cpu()
    plans = {k[-1]: p for k, p in m._plans.items() if k[0] == 1}
    assert set(plans) == {True, False}
    ws_infer, ws_train = plans[True].ws_bytes, plans[False].ws_bytes
    rel = _rel(fwd_only, train)
    print("\nC5 forward-only vs training plan (batch 1): rel-L2 %.3e, workspaces %.2f / %.2f GiB (%.1f s)"
          % (rel, ws_infer / 2 ** 30, ws_train / 2 ** 30, time.perf_counter() - t0))
    assert rel <= 1e-6
    assert ws_infer < ws_train


def test_c5_whole_volume_matches_window_by_window(pkg, oracle):
    """SlidingWindowInferer (device gather / scatter, 9 forwards of 3 tiles) against the oracle's inferer driving the same
    model one window at a time; volumetric_predictions(activation="sigmoid") returns the sigmoid of that volume"""
    t0 = time.perf_counter()
    m = _model(pkg, oracle, "bf16")
    inf = pkg.SlidingWindowInferer(roi_size=C.C5_ROI, sw_batch_size=C.C5_BATCH, overlap=C.C5_OVERLAP)
    vol = oracle["vol"]
    with torch.no_grad():
        got = inf(vol.to(DEV), m)
        ref = sliding_window_inference(vol, C.C5_ROI, lambda p: m(p.to(DEV)).cpu(), overlap=C.C5_OVERLAP)
    rel = _rel(got, ref)
    xp = vol.clone().as_subclass(_Meta)
    xp.meta = {"filename_or_obj": ["c5.nii.gz"]}
    (name, pred), = pkg.volumetric_predictions(m, [{"image": xp}], None, activation="sigmoid", inferer=inf)
    print("\nC5 256^3 volume, device inferer vs window by window: rel-L2 %.3e (%.1f s)" % (rel, time.perf_counter() - t0))
    assert rel <= 1e-6
    assert name == "c5.nii.gz"
    assert _rel(pred, torch.sigmoid(got[0])) <= 1e-6      # a second pass: only the order of the statistics atomics may differ
