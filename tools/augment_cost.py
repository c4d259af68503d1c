"""Cost of the device augmentation (augment.Compose: flips + rotation + z-score + scale + shift) per training batch.

Batches: C2 (2 x 4 x 128^3 fp32 image, 2 x 3 x 128^3 uint8 one-hot) and SPPIN (2 x 4 x 192^3 image, 2 x 1 x 192^3 label map).
The transforms are those of examples/sppin/sppin_config.json with every prob = 1, so every sample is flipped and rotated.
Timed with CUDA events after warm-up, medians of --reps:
  (a), (b) fused    augment.Compose on the batch (both passes, parameter draw and upload included)
           resample b200unet_augment_resample alone (pass 1)
  (c)      torch    a torch GPU restatement: affine_grid + grid_sample (bilinear image, nearest label) + torch z-score, scale, shift
  (d)      host     torch CPU grid_sample of ONE sample (image + label) on the host's cores: a stand-in for one loader worker's
                    per-sample resample (--host-threads sets torch's CPU threads; default 1, as in one worker)
Compulsory bytes: pass 1 reads and writes the image and the label once, pass 2 reads and writes the image; the table gives
the fused call's share of the H100 SXM data-sheet 3.35 TB/s on them.  Prints the card name and power limit of the same run.

    python tools/augment_cost.py [--reps 50] [--out FILE.json]
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dunetcnn_b200")
HBM_PEAK = 3.35e12
SPPIN = {"normalization": "NormalizeIntensityD", "normalization_kwargs": {"channel_wise": True, "nonzero": False}, "training": {
    "spatial_augmentations": [{"name": "RandFlipD", "spatial_axis": 0, "prob": 1.0}, {"name": "RandFlipD", "spatial_axis": 1, "prob": 1.0},
                              {"name": "RandRotateD", "prob": 1.0, "range_x": 0.2, "range_y": 0.2, "range_z": 0.2}],
    "intensity_augmentations": [{"name": "RandScaleIntensityD", "factors": 0.1, "prob": 1.0},
                                {"name": "RandShiftIntensityD", "offsets": 0.1, "prob": 1.0}]}}
BATCHES = {"C2": ((2, 4, 128, 128, 128), 3), "SPPIN": ((2, 4, 192, 192, 192), 1)}


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


def torch_restatement(x, lab, affine):
    """the same batch with torch ops: affine (index space, [N][3][4]) -> normalised grid, grid_sample, z-score per (n, c)"""
    n, c, d, h, w = x.shape
    size = torch.tensor([d, h, w], dtype=torch.float32, device=x.device)
    # normalised output coordinate u -> index p = ((u + 1) size - 1) / 2 -> source index A p + t -> normalised source
    s = torch.diag_embed(size / 2)
    m = torch.zeros(n, 4, 4, device=x.device)
    m[:, :3] = affine
    m[:, 3, 3] = 1
    to_idx = torch.eye(4, device=x.device).repeat(n, 1, 1)
    to_idx[:, :3, :3] = s
    to_idx[:, :3, 3] = (size - 1) / 2
    to_norm = torch.eye(4, device=x.device).repeat(n, 1, 1)
    to_norm[:, :3, :3] = torch.diag_embed(2 / size)
    to_norm[:, :3, 3] = 1 / size - 1
    theta = (to_norm @ m @ to_idx)[:, :3]
    perm = torch.tensor([2, 1, 0], device=x.device)                           # (d, h, w) -> grid's (x, y, z) = (w, h, d)
    theta = theta[:, perm][:, :, torch.cat([perm, torch.tensor([3], device=x.device)])]
    grid = F.affine_grid(theta, list(x.shape), align_corners=False)
    y = F.grid_sample(x, grid, mode="bilinear", padding_mode="border", align_corners=False)
    yl = F.grid_sample(lab.float(), grid, mode="nearest", padding_mode="border", align_corners=False).to(torch.uint8)
    mean = y.mean((2, 3, 4), keepdim=True)
    std = y.std((2, 3, 4), keepdim=True, unbiased=False)
    y = (y - mean) / torch.where(std == 0, torch.ones_like(std), std)
    return y * 1.05 + 0.02, yl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--host-threads", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "augment_cost needs a CUDA device"
    dev = torch.device("cuda")
    lib = pkg.lib.load_library()
    rows = []
    for name, (shape, nl) in BATCHES.items():
        g = torch.Generator().manual_seed(0)
        x = torch.randn(shape, generator=g).to(dev)
        lab = (torch.rand((shape[0], nl) + shape[2:], generator=g) * 2).to(torch.uint8).to(dev)
        comp, _ = pkg.augment.build_device_transform(SPPIN)
        comp.set_random_state(0)
        data = {"image": x, "label": lab}
        fused = timed(lambda: comp(data), args.reps)
        n, c, d, h, w = shape
        out, lout = torch.empty_like(x), torch.empty_like(lab)
        comp(data)
        affine = comp.last_params["affine"].float().to(dev)
        scratch = torch.empty(int(lib.b200unet_augment_scratch_bytes(n, c, d * h * w)), dtype=torch.uint8, device=dev)

        def resample():
            pkg.lib.check(lib.b200unet_augment_resample(x.data_ptr(), lab.data_ptr(), n, c, nl, d, h, w, affine.data_ptr(), 0, 0,
                                                        out.data_ptr(), lout.data_ptr(), scratch.data_ptr(), pkg.lib.stream_ptr()))
        pass1 = timed(resample, args.reps)
        ref = timed(lambda: torch_restatement(x, lab, affine), args.reps)
        # host: one sample, image + label, on the CPU
        torch.set_num_threads(args.host_threads)
        xs, ls, a1 = x[:1].cpu(), lab[:1].cpu(), affine[:1].cpu()
        ts = []
        for _ in range(args.host_reps):
            t0 = time.perf_counter()
            torch_restatement(xs, ls, a1)
            ts.append((time.perf_counter() - t0) * 1e3)
        host = statistics.median(ts)
        s = d * h * w
        byt = n * s * (4 * c * 2 + nl * 2) + n * s * 4 * c * 2
        byt1 = n * s * (4 * c * 2 + nl * 2)
        rows.append({"batch": name, "shape": list(shape), "label_channels": nl, "fused_ms": fused, "resample_ms": pass1,
                     "torch_gpu_ms": ref, "host_one_sample_ms": host, "host_threads": args.host_threads, "bytes": byt,
                     "fused_share_of_hbm": byt / (fused * 1e-3) / HBM_PEAK, "resample_share_of_hbm": byt1 / (pass1 * 1e-3) / HBM_PEAK})
    info = {"device": torch.cuda.get_device_name(), "power_limit": power_limit(), "reps": args.reps, "rows": rows}
    print("%s, power limit %s, medians of %d" % (info["device"], info["power_limit"], args.reps))
    print("| batch | (a/b) fused ms | share of HBM | pass 1 ms | (c) torch GPU ms | (d) host 1 sample ms (%d thread) |" % args.host_threads)
    for r in rows:
        print("| %s | %.3f | %.0f %% | %.3f | %.3f | %.0f |" % (r["batch"], r["fused_ms"], 100 * r["fused_share_of_hbm"], r["resample_ms"],
                                                           r["torch_gpu_ms"], r["host_one_sample_ms"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
