"""Cost of the boundary-distance metrics on the device (metrics.py), against the host path they replace.

Case: one BraTS batch 1 x 3 x 240 x 240 x 155 (three region channels), prediction and ground truth two independent draws of
lesion-like ellipsoids: small (ET-like, radii 2..6) or large (WT-like, radii 15..40).  Two calls:
  hd95       compute_hausdorff_distance(percentile=95)
  all        compute_surface_metrics: HD95 + ASD (symmetric) + NSD (tolerance 1) from one distance transform
Columns, medians of --reps after warm-up:
  call ms    CUDA events around the Python call
  kernel ms  the sum of the surface.cu kernel times in one call, from torch.profiler
  share      the bytes the passes must move (from the shapes: masks read once, W offsets 2 x 2 B written and read twice, (dh, dw)
             2 x 4 B written and read; the percentile keys of the edge voxels, a small fraction, are left out), over kernel ms,
             against the data-sheet 3.35 TB/s
  host ms    the path this replaces: device-to-host copy, then MONAI's per-(item, class, direction) scipy binary_erosion +
             distance_transform_edt and torch.quantile (tests/metrics_oracle.py), single-threaded
Prints the card name and power limit of the same run.

    python tools/metrics_cost.py [--reps 20] [--host-reps 1] [--out FILE.json]
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
pkg = importlib.import_module("3dunetcnn_b200")
HBM_PEAK = 3.35e12
SHAPE = (240, 240, 155)


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:  # noqa: BLE001
        return "unknown"


def lesions(c, n, rmin, rmax, seed, dev):
    g = torch.Generator().manual_seed(seed)
    z = torch.arange(SHAPE[0], device=dev, dtype=torch.float32).view(-1, 1, 1)
    y = torch.arange(SHAPE[1], device=dev, dtype=torch.float32).view(1, -1, 1)
    x = torch.arange(SHAPE[2], device=dev, dtype=torch.float32).view(1, 1, -1)
    out = torch.zeros((1, c) + SHAPE, dtype=torch.bool, device=dev)
    for ch in range(c):
        for _ in range(n):
            cz, cy, cx = (float(torch.randint(s // 4, 3 * s // 4, (1,), generator=g)) for s in SHAPE)
            rz, ry, rx = (float(torch.empty(1).uniform_(rmin, rmax, generator=g)) for _ in range(3))
            out[0, ch] |= ((z - cz) / rz) ** 2 + ((y - cy) / ry) ** 2 + ((x - cx) / rx) ** 2 <= 1
    return out


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
    """median over reps of the summed device time of the surface kernels in one call, their launches per call and the
    device-to-host copies per call"""
    from torch.profiler import ProfilerActivity, profile
    per, launches, d2h = [], 0, 0
    for _ in range(reps):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        t, launches, d2h = 0.0, 0, 0
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            if "k_sf_" in ev.name:
                t += ev.device_time * 1e-3
                launches += 1
            if "DtoH" in ev.name or "Device -> Pageable" in ev.name or "Device -> Pinned" in ev.name:
                d2h += 1
        per.append(t)
    return sorted(per)[len(per) // 2], launches, d2h


def host_path(P, G, q, both, reps):
    import metrics_oracle as orc
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        p, g = P.cpu().numpy(), G.cpu().numpy()
        orc.hausdorff(p, g, True, q)
        if both:
            orc.average_surface(p, g, True, True)
            orc.surface_dice(p, g, [1.0] * p.shape[1], True)
        ts.append((time.perf_counter() - t0) * 1e3)
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-reps", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/metrics_cost.py measures on a CUDA device; none is visible")
    torch.set_num_threads(1)
    dev = torch.device("cuda")
    card, plim = torch.cuda.get_device_name(dev), power_limit()
    print("card: %s, power limit %s" % (card, plim))
    M = pkg.metrics
    rows = []
    S = int(np.prod(SHAPE))
    for kind, n, rmin, rmax in (("small (ET-like)", 3, 2, 6), ("large (WT-like)", 2, 15, 40)):
        P = lesions(3, n, rmin, rmax, 1, dev)
        G = lesions(3, n, rmin, rmax, 2, dev)
        for call in ("hd95", "all"):
            if call == "hd95":
                def fn():
                    return M.compute_hausdorff_distance(P, G, include_background=True, percentile=95)
            else:
                def fn():
                    return M.compute_surface_metrics(P, G, include_background=True, percentile=95, symmetric=True,
                                                     class_thresholds=[1.0, 1.0, 1.0])
            t_call = timed(fn, a.reps, a.warmup)
            t_k, launches, d2h = kernel_ms(fn, max(3, a.reps // 4))
            V = P.shape[1]
            # compulsory bytes per pair: masks 2 x 1 B read; W offsets 2 x 2 B written, read by the H pass (the feature mask) and
            # the D pass (the query mask); (dh, dw) 2 x 4 B written and read
            moved = V * S * (2 * 1 + 2 * 2 * 3 + 2 * 4 * 2)
            row = dict(card=card, power_limit=plim, lesions=kind, call=call, call_ms=t_call, kernel_ms=t_k,
                       share=moved / HBM_PEAK / (t_k * 1e-3) if t_k > 0 else None, launches=launches, d2h_copies=d2h,
                       host_ms=host_path(P, G, 95, call == "all", a.host_reps), reps=a.reps)
            rows.append(row)
            print(json.dumps(row))
        del P, G
        torch.cuda.empty_cache()
    print("\ncard: %s, power limit %s; 1 x 3 x 240 x 240 x 155; medians of %d reps (host: %d)" % (card, plim, a.reps, a.host_reps))
    print("| lesions | call | call ms | kernel ms | share of 3.35 TB/s | launches / D2H copies | host (D2H + scipy) ms |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s | %s | %.2f | %.2f | %.0f %% | %d / %d | %.0f |" % (r["lesions"], r["call"], r["call_ms"], r["kernel_ms"],
                                                                   100 * r["share"], r["launches"], r["d2h_copies"], r["host_ms"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
