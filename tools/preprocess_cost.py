"""Cost of the training crop + resize on the device (augment.Compose with CropForegroundd + Resized ahead of the augmentation)
against the same chain on one host thread.

Batches (fp32 image, uint8 label; MRI-like: exact zeros around an N(0, 1) + 2 head region covering about a third of the volume):
  BraTS   2 x 4 x 240 x 240 x 155 + a 3-channel one-hot, foreground_percentile 0.1, to 128^3 (examples/brats2020)
  SPPIN   two sizes, 4 x 224 x 224 x 160 and 4 x 256 x 240 x 176 + a 1-channel label, foreground_percentile 0.9, to 192^3
The device Compose is the geometry stage plus the SPPIN config's flips, rotation, z-score, scale and shift (every prob = 1).
Timed with CUDA events after warm-up (medians of --reps); the per-kernel split comes from torch.profiler over --reps calls.
Compulsory bytes per kernel (share of the H100 SXM data-sheet 3.35 TB/s):
  k_fg_hist  one read of the image, per pass (3 passes)
  k_fg_box   one read of the image (the kernel stops reading a voxel's channels at the first selected one, so it may read less)
  k_aug_resample  the box of the image and the label read once, the output image and label written once
  k_aug_apply     the output image read and written
Host baseline: per sample np.percentile per channel, the mask, the box, the crop, F.interpolate trilinear (image) and nearest
(label) on one thread (torch.set_num_threads(1)), --host-reps runs of the first sample.  Also prints the extra host-to-device
bytes of shipping full-size volumes instead of resized ones.  Prints the card name and power limit of the same run.

    python tools/preprocess_cost.py [--reps 20] [--out FILE.json]
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dunetcnn_b200")
HBM_PEAK = 3.35e12
KEYS = ("image", "label")
BATCHES = {"BraTS": ([(240, 240, 155)] * 2, 3, 0.1, (128, 128, 128)),
           "SPPIN-like": ([(224, 224, 160), (256, 240, 176)], 1, 0.9, (192, 192, 192))}


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:  # noqa: BLE001
        return "unknown"


def timed(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def sample(shape, n_labels, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.zeros((4,) + shape)
    lo = [s // 5 for s in shape]
    hi = [s - s // 6 for s in shape]
    sub = tuple(b - a for a, b in zip(lo, hi))
    x[:, lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = torch.randn((4,) + sub, generator=g) + 2.0
    lab = (torch.rand((n_labels,) + shape, generator=g) > 0.7).to(torch.uint8)
    return x, lab


def host_chain(x, lab, p, out_size):
    """the reference's CropForegroundD(percentile_threshold, margin=1) + ResizeD on one sample, restated with numpy / torch"""
    a = x.numpy()
    thr = np.percentile(a.reshape(a.shape[0], -1), p * 100, axis=-1)
    mask = (a > thr[:, None, None, None]).any(0)
    box = []
    for ax in range(3):
        idx = np.nonzero(mask.any(axis=tuple(k for k in range(3) if k != ax)))[0]
        box.append((max(int(idx[0]) - 1, 0), min(int(idx[-1]) + 2, a.shape[1 + ax])))
    sl = (slice(None),) + tuple(slice(b0, b1) for b0, b1 in box)
    y = F.interpolate(x[sl][None], size=out_size, mode="trilinear", align_corners=False)
    yl = F.interpolate(lab[sl][None].float(), size=out_size, mode="nearest")
    return y, yl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "preprocess_cost needs a CUDA device"
    aug = pkg.augment
    dev = torch.device("cuda")
    rows = []
    for name, (shapes, nl, p, out_size) in BATCHES.items():
        host = [sample(s, nl, i) for i, s in enumerate(shapes)]
        data = {"image": [x.to(dev) for x, _ in host], "label": [lab.to(dev) for _, lab in host]}
        comp = aug.Compose([aug.CropForegroundd(KEYS, foreground_percentile=p), aug.Resized(KEYS, spatial_size=out_size),
                            aug.RandFlipd(KEYS, prob=1.0, spatial_axis=0), aug.RandFlipd(KEYS, prob=1.0, spatial_axis=1),
                            aug.RandRotated(KEYS, range_x=0.2, range_y=0.2, range_z=0.2, prob=1.0),
                            aug.NormalizeIntensityd("image", channel_wise=True),
                            aug.RandScaleIntensityd("image", factors=0.1, prob=1.0),
                            aug.RandShiftIntensityd("image", offsets=0.1, prob=1.0)]).set_random_state(0)
        whole = timed(lambda: comp(data), args.reps)
        box = comp.last_params["box"].cpu().numpy()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                comp(data)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            if e.device_type == torch.autograd.DeviceType.CUDA and ("k_fg_" in e.key or "k_aug_" in e.key or "memset" in e.key.lower()):
                short = next(k for k in ("k_fg_hist", "k_fg_scan", "k_fg_box", "k_fg_compose", "k_aug_resample", "k_aug_stats",
                                         "k_aug_apply", "emset") if k in e.key)
                short = "memset" if short == "emset" else short
                kern[short] = kern.get(short, 0.0) + e.device_time_total / 1e3 / args.reps      # ms per call
        c = 4
        s_in = sum(int(np.prod(s)) for s in shapes)
        s_box = sum(int(np.prod([b1 - b0 for b0, b1 in bx])) for bx in box)
        s_out = len(shapes) * int(np.prod(out_size))
        comp_bytes = {"k_fg_hist": 3 * 4 * c * s_in, "k_fg_box": 4 * c * s_in,
                      "k_aug_resample": (4 * c + nl) * s_box + (4 * c + nl) * s_out, "k_aug_apply": 2 * 4 * c * s_out}
        share = {k: comp_bytes[k] / (kern[k] * 1e-3) / HBM_PEAK for k in comp_bytes if kern.get(k)}
        torch.set_num_threads(1)
        ts = []
        for _ in range(args.host_reps):
            t0 = time.perf_counter()
            host_chain(host[0][0], host[0][1], p, out_size)
            ts.append(time.perf_counter() - t0)
        rows.append({"batch": name, "shapes": [list(s) for s in shapes], "label_channels": nl, "percentile": p,
                     "out": list(out_size), "compose_ms": whole, "kernels_ms": kern, "compulsory_bytes": comp_bytes,
                     "share_of_hbm": share, "host_one_sample_s": statistics.median(ts),
                     "h2d_image_bytes_per_sample_raw": 4 * c * int(np.prod(shapes[0])),
                     "h2d_image_bytes_per_sample_resized": 4 * c * int(np.prod(out_size)),
                     "h2d_label_bytes_per_sample_raw": nl * int(np.prod(shapes[0])),
                     "h2d_label_bytes_per_sample_resized": nl * int(np.prod(out_size))})
    info = {"device": torch.cuda.get_device_name(), "power_limit": power_limit(), "reps": args.reps, "rows": rows}
    print("%s, power limit %s, medians of %d" % (info["device"], info["power_limit"], args.reps))
    for r in rows:
        print("%s %s -> %s: Compose %.3f ms per batch; host chain %.2f s per sample (1 thread); image H2D per sample %.1f MB raw "
              "vs %.1f MB resized" % (r["batch"], r["shapes"], r["out"], r["compose_ms"], r["host_one_sample_s"],
                                      r["h2d_image_bytes_per_sample_raw"] / 1e6, r["h2d_image_bytes_per_sample_resized"] / 1e6))
        for k, v in sorted(r["kernels_ms"].items(), key=lambda kv: -kv[1]):
            sh = r["share_of_hbm"].get(k)
            print("   %-15s %.3f ms%s" % (k, v, "  %.0f %% of 3.35 TB/s" % (100 * sh) if sh is not None else ""))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
