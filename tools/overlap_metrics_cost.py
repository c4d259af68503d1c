"""Cost of the overlap metrics on the device (metrics.py: DiceHelper / compute_dice, one counting pass of overlap.cu), against a
torch restatement of MONAI's path on the same GPU.

Cases (seeded random inputs):
  brats       1 x 3 x 240 x 240 x 155, sigmoid logits (fp32) against a uint8 one-hot target
  c2          2 x 3 x 128^3, sigmoid logits against a uint8 one-hot target
  c104        2 x 104 x 128^3, argmax of fp32 logits against a uint8 label map
  c104_maps   2 x 1 x 128^3, a uint8 label map of 104 classes against a uint8 label map
Columns, medians of --reps after warm-up:
  call ms     CUDA events around DiceHelper(...)(y_pred, y) (per-pair Dice, reduction "none"): the counting launch and the torch
              ops on the [B, C] counts
  kernel ms   k_overlap_counts alone, from torch.profiler
  share       the bytes the pass must read (every input byte once), over kernel ms, against the data-sheet 3.35 TB/s
  torch ms    MONAI's path restated in torch on the device: sigmoid and threshold, or argmax and a one-hot expansion (a broadcast
              compare to a bool [B, C, ...] tensor, of the label-map target too), then per-class sums of I, P and G
Prints the card name and power limit of the same run.

    python tools/overlap_metrics_cost.py [--reps 20] [--out FILE.json]
"""
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
HBM_PEAK = 3.35e12
CASES = [("brats", 1, 3, (240, 240, 155), "sigmoid"), ("c2", 2, 3, (128, 128, 128), "sigmoid"),
         ("c104", 2, 104, (128, 128, 128), "argmax"), ("c104_maps", 2, 104, (128, 128, 128), "labels")]


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:  # noqa: BLE001
        return "unknown"


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def kernel_ms(fn, reps):
    """median over reps of the device time of k_overlap_counts in one call"""
    from torch.profiler import ProfilerActivity, profile
    per = []
    for _ in range(reps):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        per.append(sum(ev.device_time * 1e-3 for ev in prof.events()
                       if ev.device_type == torch.autograd.DeviceType.CUDA and "k_overlap_counts" in ev.name))
    return sorted(per)[len(per) // 2]


def inputs(kind, b, c, shape, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    if kind == "labels":
        pred = torch.randint(0, c, (b, 1) + shape, generator=g, device=dev, dtype=torch.uint8)
    else:
        pred = torch.randn((b, c) + shape, generator=g, device=dev)
    if kind == "sigmoid":
        y = (torch.rand((b, c) + shape, generator=g, device=dev) < 0.3).to(torch.uint8)
    else:
        y = torch.randint(0, c, (b, 1) + shape, generator=g, device=dev, dtype=torch.uint8)
    return pred, y


def torch_path(kind, c, pred, y):
    """MONAI's steps in torch: discretise, expand to one-hot, sum per class.  (P, G, I) int64 [B, C]"""
    dims = (2, 3, 4)
    cls = torch.arange(c, device=pred.device, dtype=torch.int64).view(1, c, 1, 1, 1)
    if kind == "sigmoid":
        p, t = torch.sigmoid(pred) > 0.5, y.bool()
    else:
        lab = torch.argmax(pred, dim=1, keepdim=True) if kind == "argmax" else pred.long()
        p, t = lab == cls, y.long() == cls
    return p.sum(dims), t.sum(dims), (p & t).sum(dims)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/overlap_metrics_cost.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda")
    card, plim = torch.cuda.get_device_name(dev), power_limit()
    print("card: %s, power limit %s" % (card, plim))
    M = pkg.metrics
    rows = []
    for name, b, c, shape, kind in CASES:
        pred, y = inputs(kind, b, c, shape, dev)
        if kind == "sigmoid":
            helper = M.DiceHelper(sigmoid=True, activate=True, include_background=True, reduction="none", get_not_nans=False)
        else:
            helper = M.DiceHelper(softmax=kind == "argmax", include_background=True, reduction="none", get_not_nans=False,
                                  num_classes=c)
        got = torch.stack(helper.counts(pred, y))
        ref = torch.stack(torch_path(kind, c, pred, y))
        assert torch.equal(got, ref), "counts differ from the torch restatement"
        t_call = timed(lambda: helper(pred, y), a.reps, a.warmup)
        t_k = kernel_ms(lambda: helper(pred, y), max(3, a.reps // 4))
        t_torch = timed(lambda: torch_path(kind, c, pred, y), a.reps, a.warmup)
        moved = pred.numel() * pred.element_size() + y.numel() * y.element_size()
        row = dict(card=card, power_limit=plim, case=name, shape=[b, c] + list(shape), pred=kind, bytes=moved, call_ms=t_call,
                   kernel_ms=t_k, share=moved / HBM_PEAK / (t_k * 1e-3) if t_k > 0 else None, torch_ms=t_torch, reps=a.reps)
        rows.append(row)
        print(json.dumps(row))
        del pred, y, got, ref
        torch.cuda.empty_cache()
    print("\ncard: %s, power limit %s; medians of %d reps" % (card, plim, a.reps))
    print("| case | B x C x D x H x W | prediction | MB read | call ms | kernel ms | share of 3.35 TB/s | torch restatement ms |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s | %s | %s | %.1f | %.3f | %.3f | %.0f %% | %.3f |" % (r["case"], " x ".join(map(str, r["shape"])), r["pred"],
                                                                         r["bytes"] / 1e6, r["call_ms"], r["kernel_ms"],
                                                                         100 * r["share"], r["torch_ms"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
