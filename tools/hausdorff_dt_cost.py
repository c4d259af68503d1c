"""Cost of HausdorffDTLoss on the device (losses.py, csrc/hausdorff_dt.cu + csrc/dice_ce.cu), against the host path it replaces.

Cases (logits and targets are smooth random blobs, so the masks have the extents of organs rather than of voxel noise):
  C2        2 x 3 x 128^3, sigmoid, uint8 one-hot target
  16-class  2 x 16 x 128^3, softmax, uint8 label map (to_onehot_y)
  BraTS     1 x 3 x 240 x 240 x 155, sigmoid, uint8 one-hot region target, include_background=True
Columns, medians of --reps after warm-up:
  fwd ms / bwd ms   CUDA events around the criterion call and around loss.backward()
  kernel ms         each kernel's device time in one forward + backward, from torch.profiler in a run of its own
  share             the bytes the kernel must move (from the shapes: the logits, the target bytes it reads, the 8 B of W offsets
                    and 16 B of (dh, dw) per kept (n, c) and voxel, the 4 B weight, dlogits), over its time, against the
                    data-sheet 3.35 TB/s
  host ms           the path this replaces, MONAI's: a device-to-host copy of the activated prediction and the target, then
                    scipy's distance_transform_edt of the mask and of its complement, for the prediction and the target of every
                    kept (n, c), on one thread (the loss arithmetic after it is left out)
Prints the card name and power limit of the same run.

    python tools/hausdorff_dt_cost.py [--reps 20] [--host-reps 1] [--cases C2,16-class,BraTS] [--out FILE.json]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F
from scipy.ndimage import distance_transform_edt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dunetcnn_b200")
HBM_PEAK = 3.35e12
CASES = [
    # name, n, c, spatial, act, target form, include_background
    ("C2", 2, 3, (128, 128, 128), "sigmoid", "onehot_u8", False),
    ("16-class", 2, 16, (128, 128, 128), "softmax", "label_u8", False),
    ("BraTS", 1, 3, (240, 240, 155), "sigmoid", "onehot_u8", True),
]
KERNELS = ("k_hd_rows", "k_hd_cols_h", "k_hd_cols_d", "k_dice_ce_fwd", "k_dice_ce_reduce", "k_dice_finalize", "k_dice_ce_bwd")


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:  # noqa: BLE001
        return "unknown"


def blobs(shape, seed, dev):
    """smooth random fields: noise on a grid 8x coarser, trilinearly up-sampled"""
    g = torch.Generator(device=dev).manual_seed(seed)
    coarse = torch.randn(shape[:2] + tuple(max(2, s // 8) for s in shape[2:]), generator=g, device=dev)
    return F.interpolate(coarse, size=shape[2:], mode="trilinear", align_corners=False)


def inputs(n, c, spatial, form, seed, dev):
    x = 3.0 * blobs((n, c) + spatial, seed, dev)
    field = blobs((n, c) + spatial, seed + 1, dev)
    if form == "label_u8":
        return x, field.argmax(1, keepdim=True).to(torch.uint8)
    return x, (field > 0.3).to(torch.uint8)


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def kernel_ms(step, reps):
    """per kernel: the median over reps of its device time in one forward + backward, its launches per step, and the names of
    the device kernels the profiler recorded in the last rep"""
    from torch.profiler import ProfilerActivity, profile
    per = {k: [] for k in KERNELS}
    launches = {k: 0 for k in KERNELS}
    for _ in range(reps):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        t = {k: 0.0 for k in KERNELS}
        launches = {k: 0 for k in KERNELS}
        seen = set()
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            seen.add(ev.name[:60])
            for k in KERNELS:
                if k in ev.name:
                    t[k] += ev.device_time * 1e-3
                    launches[k] += 1
        for k in KERNELS:
            per[k].append(t[k])
    return {k: sorted(v)[len(v) // 2] for k, v in per.items()}, launches, sorted(seen)


def kernel_bytes(n, c, s, act, form, kept):
    """bytes each kernel must move"""
    v = n * kept * s
    tb = n * s if form == "label_u8" else n * c * s            # the loss kernels stage every channel of a one-hot target
    tb_rows = n * s if form == "label_u8" else v               # the row pass reads the kept channels only
    logits_rows = 4 * n * c * s if act == "softmax" else 4 * v
    return {
        "k_hd_rows": logits_rows + tb_rows + 8 * v,
        "k_hd_cols_h": 8 * v + 16 * v,
        "k_hd_cols_d": 16 * v + 8 * v + 4 * v,
        "k_dice_ce_fwd": 4 * n * c * s + tb + 4 * v,
        "k_dice_ce_bwd": 4 * n * c * s + tb + 4 * v + 4 * n * c * s,
    }


def host_path(x, t, act, c, include_background, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        p = (torch.sigmoid(x) if act == "sigmoid" else torch.softmax(x, 1)).cpu().numpy()
        tt = t.cpu().numpy()
        if tt.shape[1] == 1:
            tt = np.stack([tt[:, 0] == k for k in range(c)], 1)
        lo = 0 if include_background else 1
        for n in range(p.shape[0]):
            for k in range(lo, c):
                for m in (p[n, k] > 0.5, tt[n, k] > 0.5):
                    if m.any() and not m.all():
                        distance_transform_edt(m)
                        distance_transform_edt(~m)
        ts.append((time.perf_counter() - t0) * 1e3)
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-reps", type=int, default=1)
    ap.add_argument("--cases", default=",".join(c[0] for c in CASES))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/hausdorff_dt_cost.py measures on a CUDA device; none is visible")
    torch.set_num_threads(1)
    dev = torch.device("cuda")
    card, plim = torch.cuda.get_device_name(dev), power_limit()
    print("card: %s, power limit %s" % (card, plim))
    rows = []
    for name, n, c, spatial, act, form, ib in CASES:
        if name not in a.cases.split(","):
            continue
        x, t = inputs(n, c, spatial, form, 7, dev)
        crit = pkg.HausdorffDTLoss(sigmoid=act == "sigmoid", softmax=act == "softmax", to_onehot_y=form == "label_u8",
                                   include_background=ib)
        xx = x.clone().requires_grad_(True)
        state = {}

        def fwd():
            state["loss"] = crit(xx, t)

        def bwd():
            state["loss"].backward()

        def step():
            crit(xx, t).backward()

        for _ in range(a.warmup):
            step()
        t_f, t_b = [], []
        for _ in range(a.reps):
            t_f.append(timed(fwd, 1, 0))
            t_b.append(timed(bwd, 1, 0))
        t_f, t_b = sorted(t_f)[len(t_f) // 2], sorted(t_b)[len(t_b) // 2]
        per, launches, seen = kernel_ms(step, max(3, a.reps // 4))
        s = int(np.prod(spatial))
        kept = c if ib else c - 1
        moved = kernel_bytes(n, c, s, act, form, kept)
        share = {k: (moved[k] / HBM_PEAK / (per[k] * 1e-3) if k in moved and per[k] > 0 else None) for k in KERNELS}
        row = dict(card=card, power_limit=plim, case=name, shape=[n, c] + list(spatial), act=act, target=form, fwd_ms=t_f, bwd_ms=t_b,
                   kernel_ms=per, launches=launches, profiled=seen, share=share, host_ms=host_path(x, t, act, c, ib, a.host_reps), reps=a.reps)
        rows.append(row)
        print(json.dumps(row))
        del x, t, xx, state
        torch.cuda.empty_cache()
    print("\ncard: %s, power limit %s; medians of %d reps (host: %d)" % (card, plim, a.reps, a.host_reps))
    print("| case | fwd ms | bwd ms | rows | cols H | cols D | loss fwd | loss bwd | host (D2H + scipy) ms |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        cells = []
        for k in ("k_hd_rows", "k_hd_cols_h", "k_hd_cols_d", "k_dice_ce_fwd", "k_dice_ce_bwd"):
            cells.append("%.2f (%.0f %%)" % (r["kernel_ms"][k], 100 * (r["share"][k] or 0)))
        print("| %s %s | %.2f | %.2f | %s | %.0f |" % (r["case"], "x".join(map(str, r["shape"])), r["fwd_ms"], r["bwd_ms"],
                                                      " | ".join(cells), r["host_ms"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
