"""Throughput of one SegResNet training step (forward + sigmoid Dice + backward + fused Adam) through the plan, eager and as a
CUDA-graph replay, next to the same step of the oracle's torch restatement (oracle/segresnet_oracle.py) under bf16 autocast with
cudnn.benchmark, on the same GPU in the same call.  One JSON line per workload:
  brats:  MONAI's BraTS recipe -- init_filters 16, blocks_down [1, 2, 2, 4], blocks_up [1, 1, 1], 4 -> 3 channels, dropout 0.2 --
          batch 1 at 224 x 224 x 144
  c2:     the same network, batch 2 at 4 x 128^3
Usage: python tools/segresnet_bench.py [--workloads brats,c2] [--reps 5]"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dunetcnn_b200")
from oracle.segresnet_oracle import segresnet_forward  # noqa: E402

KW = dict(init_filters=16, in_channels=4, out_channels=3, dropout_prob=0.2, blocks_down=[1, 2, 2, 4], blocks_up=[1, 1, 1])
WORKLOADS = {"brats": (1, (224, 224, 144)), "c2": (2, (128, 128, 128))}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(q.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001
        power = None
    return name, power


def timeit(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        loss = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, float(loss)


def sigmoid_dice(logits, t):
    p = torch.sigmoid(logits.float())
    dims = tuple(range(2, p.dim()))
    i = (p * t).sum(dims)
    return (1 - (2 * i + 1e-5) / (p.sum(dims) + t.sum(dims) + 1e-5)).mean()


def run(name, reps):
    n, dims = WORKLOADS[name]
    torch.manual_seed(0)
    x = torch.randn(n, 4, *dims, device="cuda")
    t = (torch.rand(n, 3, *dims, device="cuda") > 0.7).to(torch.uint8)
    model = pkg.SegResNet(precision="bf16", **KW).cuda().train()
    crit = pkg.DiceLoss(sigmoid=True)
    opt = torch.optim.Adam(model.parameters(), lr=1e-4, fused=True)

    def eager():
        opt.zero_grad(set_to_none=True)
        loss = crit(model(x), t)
        loss.backward()
        opt.step()
        return loss
    ms_e, loss_e = timeit(eager, reps)
    launches = model.launches_last_forward + model.launches_last_backward
    plan = model._plan_for(x)
    flops = 2.0 * sum(plan.algorithmic_macs().values())
    plan.profile_begin(8192)
    eager()
    torch.cuda.synchronize()
    prof = {k: round(v["ms"], 3) for k, v in plan.profile_end().items()}
    out = {"workload": name, "model": "SegResNet", "kw": KW, "batch": n, "shape": [4, *dims], "eager_ms_per_step": ms_e,
           "eager_volumes_per_s": n / (ms_e / 1e3), "loss": loss_e, "algorithmic_tflop_per_step": flops / 1e12,
           "tflops_eager": flops / (ms_e / 1e3) / 1e12, "profile_ms": prof, "launches": launches, "workspace_gb": plan.ws_bytes / 2 ** 30}
    try:
        step = pkg.train.GraphedTrainStep(model, crit, opt, x.shape, t.shape)
        ms_g, _ = timeit(lambda: step(x, t), reps)
        out.update(graph_ms_per_step=ms_g, graph_volumes_per_s=n / (ms_g / 1e3), tflops_graph=flops / (ms_g / 1e3) / 1e12)
    except Exception as e:  # noqa: BLE001
        out["graph_error"] = repr(e)[:200]
    del model, opt, plan
    torch.cuda.empty_cache()

    # the oracle's torch restatement under bf16 autocast, cuDNN autotuned
    torch.backends.cudnn.benchmark = True
    sd = {k: v.detach().cuda().requires_grad_(True) for k, v in pkg.SegResNet(**KW).state_dict().items()}
    opt_t = torch.optim.Adam(list(sd.values()), lr=1e-4, fused=True)
    tf = t.float()

    def torch_step():
        opt_t.zero_grad(set_to_none=True)
        keep = (torch.rand(n, KW["init_filters"], device="cuda") >= KW["dropout_prob"]).float() / (1 - KW["dropout_prob"])
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits = segresnet_forward(sd, x, KW["blocks_down"], KW["blocks_up"], 8, keep)
        loss = sigmoid_dice(logits, tf)
        loss.backward()
        opt_t.step()
        return loss
    try:
        ms_t, _ = timeit(torch_step, reps)
        out.update(torch_autocast_ms_per_step=ms_t, torch_autocast_volumes_per_s=n / (ms_t / 1e3),
                   speedup_graph_vs_torch=ms_t / out.get("graph_ms_per_step", ms_e), speedup_eager_vs_torch=ms_t / ms_e)
    except Exception as e:  # noqa: BLE001
        out["torch_error"] = repr(e)[:200]
    del sd, opt_t
    torch.cuda.empty_cache()
    out["gpu"], out["power_limit_w"] = card()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="brats,c2")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    for w in a.workloads.split(","):
        run(w, a.reps)


if __name__ == "__main__":
    main()
