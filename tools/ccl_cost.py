"""Cost of connected-component post-processing on the device, against the host path it replaces.

Shapes: 1 x 256^3 and 3 x 256^3 (the three BraTS channels cleaned independently).  Masks: blobs (union of 40 balls per volume)
and Bernoulli noise at p = 0.25, at connectivity 1 and 3.  Timed with CUDA events after warm-up, medians of --reps:
  label      b200unet_cc_label alone (raster numbering, counts, sizes)
  sort       b200unet_cc_sort_by_size alone
  cc         prepost.connected_components, end to end (both calls and the read-back of the counts)
  keep       prepost.keep_largest_connected_component on the fp32 one-hot image (independent channels, num_components 1)
  host       the path this replaces: device-to-host copy of the fp32 prediction, then scipy.ndimage.label and a stable size
             ranking per volume (reported as absent when scipy is not installed)
Compulsory traffic is 1 B of mask read + 4 B of labels written per voxel; the table gives the labelling's rate against the
H100 SXM data-sheet 3.35 TB/s on those bytes.  Prints the card name and power limit of the same run.

    python tools/ccl_cost.py [--reps 10] [--size 256] [--out FILE.json]
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
pkg = importlib.import_module("3dunetcnn_b200")
HBM_PEAK = 3.35e12


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:  # noqa: BLE001
        return "unknown"


def blobs(n, size, seed, dev):
    g = torch.Generator().manual_seed(seed)
    z = torch.arange(size, device=dev).view(-1, 1, 1)
    y = torch.arange(size, device=dev).view(1, -1, 1)
    x = torch.arange(size, device=dev).view(1, 1, -1)
    out = torch.zeros((n, size, size, size), dtype=torch.bool, device=dev)
    for v in range(n):
        for _ in range(40):
            c = torch.randint(0, size, (3,), generator=g).tolist()
            r = int(torch.randint(4, 31, (1,), generator=g))
            out[v] |= (z - c[0]) ** 2 + (y - c[1]) ** 2 + (x - c[2]) ** 2 <= r * r
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


def host_path(pred, conn, reps):
    try:
        from scipy import ndimage
    except ImportError:
        return None
    st = ndimage.generate_binary_structure(3, conn)
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        p = pred.cpu().numpy()
        for v in range(p.shape[0]):
            lab, k = ndimage.label(p[v] > 0.5, structure=st)
            sizes = np.bincount(lab.ravel(), minlength=k + 1)[1:]
            order = np.argsort(-sizes, kind="stable")
            newlab = np.zeros(k + 1, np.int32)
            newlab[order + 1] = np.arange(1, k + 1, dtype=np.int32)
            newlab[lab]
        ts.append((time.perf_counter() - t0) * 1e3)
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/ccl_cost.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda")
    card, plim = torch.cuda.get_device_name(dev), power_limit()
    print("card: %s, power limit %s" % (card, plim))
    L = pkg.lib
    rows = []
    for nvol in (1, 3):
        for kind in ("blobs", "noise25"):
            if kind == "blobs":
                fg = blobs(nvol, a.size, 100 + nvol, dev)
            else:
                g = torch.Generator(device=dev).manual_seed(200 + nvol)
                fg = torch.rand((nvol,) + (a.size,) * 3, device=dev, generator=g) < 0.25
            pred = fg.float() * 0.8 + 0.1                   # an fp32 "probability" whose > 0.5 is the mask
            m8 = fg.view(torch.uint8)
            img = torch.cat([torch.zeros_like(pred[:1]), fg.float()])           # one-hot image: background + nvol channels
            for conn in (1, 3):
                d = h = w = a.size
                labels = torch.empty(m8.shape, dtype=torch.int32, device=dev)
                counts = torch.empty(nvol, dtype=torch.int32, device=dev)
                scratch = torch.empty(L.cc_scratch_bytes(nvol, d, h, w), dtype=torch.uint8, device=dev)
                L.cc_label(m8, conn, labels, counts, scratch)
                kmax = int(counts.max())

                def sort_only():
                    L.cc_label(m8, conn, labels, counts, scratch)       # the sort consumes the sizes: relabel first ...
                    e.record()                                          # ... and time from here
                    L.cc_sort_by_size(labels, kmax, scratch)

                t_label = timed(lambda: L.cc_label(m8, conn, labels, counts, scratch), a.reps, a.warmup)
                sort_ts = []
                for rep in range(a.warmup + a.reps):
                    e, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    sort_only()
                    e1.record()
                    torch.cuda.synchronize()
                    if rep >= a.warmup:
                        sort_ts.append(e.elapsed_time(e1))
                t_sort = sorted(sort_ts)[len(sort_ts) // 2]
                t_cc = timed(lambda: pkg.prepost.connected_components(m8, connectivity=conn), a.reps, a.warmup)
                t_keep = timed(lambda: pkg.prepost.keep_largest_connected_component(img, connectivity=conn), a.reps, a.warmup)
                t_host = host_path(pred, conn, a.host_reps)
                vox = nvol * d * h * w
                row = dict(card=card, power_limit=plim, volumes=nvol, size=a.size, mask=kind, connectivity=conn, max_components=kmax,
                           label_ms=t_label, sort_ms=t_sort, connected_components_ms=t_cc, keep_largest_ms=t_keep,
                           host_ms=t_host, label_compulsory_share=5 * vox / HBM_PEAK / (t_label * 1e-3), reps=a.reps)
                rows.append(row)
                print(json.dumps(row))
                del labels, counts, scratch
            del fg, pred, m8, img
            torch.cuda.empty_cache()
    print("\ncard: %s, power limit %s; %d^3 voxels per volume; medians of %d reps (host: %d)" % (card, plim, a.size, a.reps, a.host_reps))
    print("| volumes | mask | conn | K (max) | label ms | sort ms | connected_components ms | keep_largest ms | host (D2H + scipy) ms |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        host = "absent (no scipy)" if r["host_ms"] is None else "%.0f" % r["host_ms"]
        print("| %d | %s | %d | %d | %.2f | %.2f | %.2f | %.2f | %s |" % (r["volumes"], r["mask"], r["connectivity"], r["max_components"],
                                                                    r["label_ms"], r["sort_ms"], r["connected_components_ms"],
                                                                    r["keep_largest_ms"], host))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
