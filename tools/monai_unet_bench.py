"""Time of one MONAI UNet training step (forward + DiceCELoss(softmax=True, to_onehot_y=True) + backward + fused Adam) through the
plan, eager and as a CUDA-graph replay, next to the same step of the oracle's torch restatement (oracle/unet_oracle.py) under bf16
autocast with cudnn.benchmark, on the same GPU in the same call.  Each variant is timed over --windows windows of --reps steps
(CUDA events around each window, after a warm-up); the JSON line per workload gives the mean, min and max ms per step.
  spleen:  MONAI's spleen tutorial network -- channels (16, 32, 64, 128, 256), strides 2, num_res_units 2, PReLU, instance
           norm -- 1 -> 2 channels, batch 4 at 96^3
  brats:   the same network, 4 -> 3 channels, batch 2 at 128^3
Usage: python tools/monai_unet_bench.py [--workloads spleen,brats] [--reps 10] [--windows 5]"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dunetcnn_b200")
from oracle.unet_oracle import MonaiUNetConfig, unet_forward  # noqa: E402

CHANNELS = (16, 32, 64, 128, 256)
WORKLOADS = {"spleen": (4, 1, 2, (96, 96, 96)), "brats": (2, 4, 3, (128, 128, 128))}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(q.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001
        power = None
    return name, power


def timeit(fn, reps, windows):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            loss = fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / reps)
    return {"mean": sum(ms) / len(ms), "min": min(ms), "max": max(ms)}, float(loss.detach())


def dice_ce(logits, label):
    """MONAI DiceCELoss(softmax=True, to_onehot_y=True) with its defaults: mean soft Dice (smooth 1e-5) + mean cross-entropy"""
    logits = logits.float()
    onehot = F.one_hot(label[:, 0].long(), logits.shape[1]).movedim(-1, 1).float()
    p = torch.softmax(logits, 1)
    dims = tuple(range(2, p.dim()))
    i = (p * onehot).sum(dims)
    dice = (1 - (2 * i + 1e-5) / (p.sum(dims) + onehot.sum(dims) + 1e-5)).mean()
    return dice + F.cross_entropy(logits, label[:, 0].long())


def run(name, reps, windows):
    n, cin, cout, dims = WORKLOADS[name]
    kw = dict(in_channels=cin, out_channels=cout, channels=CHANNELS, strides=(2, 2, 2, 2), num_res_units=2)
    torch.manual_seed(0)
    x = torch.randn(n, cin, *dims, device="cuda")
    t = torch.randint(0, cout, (n, 1, *dims), device="cuda", dtype=torch.uint8)
    model = pkg.UNet(precision="bf16", **kw).cuda().train()
    crit = pkg.DiceCELoss(softmax=True, to_onehot_y=True)
    opt = torch.optim.Adam(model.parameters(), lr=1e-4, fused=True)

    def eager():
        opt.zero_grad(set_to_none=True)
        loss = crit(model(x), t)
        loss.backward()
        opt.step()
        return loss
    ms_e, loss_e = timeit(eager, reps, windows)
    launches = model.launches_last_forward + model.launches_last_backward
    plan = model._plan_for(x)
    flops = 2.0 * sum(plan.algorithmic_macs().values())
    plan.profile_begin(8192)
    eager()
    torch.cuda.synchronize()
    prof = {k: round(v["ms"], 3) for k, v in plan.profile_end().items()}
    out = {"workload": name, "model": "UNet", "kw": kw, "batch": n, "shape": [cin, *dims], "reps": reps, "windows": windows,
           "eager_ms_per_step": ms_e, "loss": loss_e, "algorithmic_tflop_per_step": flops / 1e12,
           "tflops_eager": flops / (ms_e["mean"] / 1e3) / 1e12, "profile_ms": prof, "launches": launches,
           "workspace_gb": plan.ws_bytes / 2 ** 30}
    try:
        step = pkg.train.GraphedTrainStep(model, crit, opt, x.shape, t.shape)
        ms_g, _ = timeit(lambda: step(x, t), reps, windows)
        out.update(graph_ms_per_step=ms_g, graph_volumes_per_s=n / (ms_g["mean"] / 1e3), tflops_graph=flops / (ms_g["mean"] / 1e3) / 1e12)
    except Exception as e:  # noqa: BLE001
        out["graph_error"] = repr(e)[:200]
    del model, opt, plan
    torch.cuda.empty_cache()

    # the oracle's torch restatement under bf16 autocast, cuDNN autotuned
    torch.backends.cudnn.benchmark = True
    cfg = MonaiUNetConfig(cin, cout, CHANNELS, 2, "prelu")
    sd = {k: v.detach().cuda().requires_grad_(True) for k, v in pkg.UNet(**kw).state_dict().items()}
    opt_t = torch.optim.Adam(list(sd.values()), lr=1e-4, fused=True)

    def torch_step():
        opt_t.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits = unet_forward(x, sd, cfg)
        loss = dice_ce(logits, t)
        loss.backward()
        opt_t.step()
        return loss
    try:
        ms_t, _ = timeit(torch_step, reps, windows)
        out.update(torch_autocast_ms_per_step=ms_t, speedup_graph_vs_torch=ms_t["mean"] / out.get("graph_ms_per_step", ms_e)["mean"],
                   speedup_eager_vs_torch=ms_t["mean"] / ms_e["mean"])
    except Exception as e:  # noqa: BLE001
        out["torch_error"] = repr(e)[:200]
    del sd, opt_t
    torch.cuda.empty_cache()
    out["gpu"], out["power_limit_w"] = card()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="spleen,brats")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--windows", type=int, default=5)
    a = ap.parse_args()
    for w in a.workloads.split(","):
        run(w, a.reps, a.windows)


if __name__ == "__main__":
    main()
