"""Cost of the segmentation criteria by class count at the C2 size (2 x 128^3 voxels, fp32 NCDHW logits).

For each C, four criteria, forward and backward timed separately with CUDA events, after warm-up, the criteria alternating
within every repetition:
  (a) DiceLoss(sigmoid=True) on a uint8 one-hot target      (the criterion the package offered before DiceCELoss)
  (b) DiceCELoss(softmax=True, to_onehot_y=True) on a uint8 label map
  (c) the same with lambda_ce = 0                             (softmax Dice alone)
  (d) tests/dice_ce_oracle.py's torch-op restatement of (b), fp32 on the same GPU
For the fused criteria it reports the HBM bytes each direction needs (computed from shapes: logits, target, dlogits), the
achieved share of the H100 SXM data-sheet 3.35 TB/s, and the host-to-device target bytes per batch of both target forms.
Prints the card name and power limit of the same run.

    python tools/loss_cost.py [--reps 20] [--classes 3,16,32,64,104,128] [--out FILE.json]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
pkg = importlib.import_module("3dunetcnn_b200")
from dice_ce_oracle import dice_ce_loss  # noqa: E402

HBM_PEAK = 3.35e12
N, S = 2, 128


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:  # noqa: BLE001
        return "unknown"


def fused_bytes(c, vox, target_bytes_per_voxel):
    """forward: logits + target read once; backward: logits + target read once, dlogits written once"""
    return vox * (4 * c + target_bytes_per_voxel), vox * (8 * c + target_bytes_per_voxel)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--classes", default="3,16,32,64,104,128")
    ap.add_argument("--size", type=int, default=S)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/loss_cost.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda")
    card = torch.cuda.get_device_name(dev)
    plim = power_limit()
    print("card: %s, power limit %s" % (card, plim))
    vox = N * a.size ** 3
    rows = []
    for c in [int(v) for v in a.classes.split(",")]:
        g = torch.Generator(device=dev).manual_seed(c)
        x = torch.randn((N, c) + (a.size,) * 3, device=dev, generator=g)
        lab = torch.randint(0, c, (N, 1) + (a.size,) * 3, device=dev, generator=g).to(torch.uint8)
        onehot = torch.nn.functional.one_hot(lab[:, 0].long(), c).movedim(-1, 1).to(torch.uint8).contiguous()
        crits = {
            "a": (pkg.DiceLoss(sigmoid=True), onehot),
            "b": (pkg.DiceCELoss(softmax=True, to_onehot_y=True), lab),
            "c": (pkg.DiceCELoss(softmax=True, to_onehot_y=True, lambda_ce=0.0), lab),
            "d": (lambda o, t: dice_ce_loss(o, t, softmax=True), lab),
        }
        times = {k: ([], []) for k in crits}
        for rep in range(a.warmup + a.reps):
            for k, (crit, t) in crits.items():
                xx = x.detach().requires_grad_(True)
                e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                e0.record()
                loss = crit(xx, t)
                e1.record()
                loss.backward()
                e2.record()
                torch.cuda.synchronize()
                if rep >= a.warmup:
                    times[k][0].append(e0.elapsed_time(e1))
                    times[k][1].append(e1.elapsed_time(e2))
                del loss, xx
        med = {k: (sorted(f)[len(f) // 2], sorted(b)[len(b) // 2]) for k, (f, b) in times.items()}
        fb_a = fused_bytes(c, vox, c)          # (a): uint8 one-hot target, C bytes per voxel
        fb_b = fused_bytes(c, vox, 1)          # (b), (c): uint8 label map, 1 byte per voxel
        row = dict(classes=c, voxels=vox, card=card, power_limit=plim, reps=a.reps,
                   h2d_target_bytes_onehot_u8=vox * c, h2d_target_bytes_label_u8=vox)
        for k in crits:
            row["%s_fwd_ms" % k], row["%s_bwd_ms" % k] = med[k]
            row["%s_total_ms" % k] = med[k][0] + med[k][1]
        for k, fb in (("a", fb_a), ("b", fb_b), ("c", fb_b)):
            row["%s_fwd_bytes" % k], row["%s_bwd_bytes" % k] = fb
            row["%s_fwd_hbm_share" % k] = fb[0] / HBM_PEAK / (med[k][0] * 1e-3)
            row["%s_bwd_hbm_share" % k] = fb[1] / HBM_PEAK / (med[k][1] * 1e-3)
        rows.append(row)
        print(json.dumps(row))
        del x, lab, onehot, crits
        torch.cuda.empty_cache()
    print("\ncard: %s, power limit %s; 2 x %d^3 voxels; medians of %d reps" % (card, plim, a.size, a.reps))
    print("| C | (a) fwd / bwd ms | (b) fwd / bwd ms | (b) HBM share fwd / bwd | (c) fwd / bwd ms | (d) fwd / bwd ms | target H2D one-hot / label map |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %d | %.3f / %.3f | %.3f / %.3f | %.0f %% / %.0f %% | %.3f / %.3f | %.2f / %.2f | %.1f MB / %.1f MB |"
              % (r["classes"], r["a_fwd_ms"], r["a_bwd_ms"], r["b_fwd_ms"], r["b_bwd_ms"], 100 * r["b_fwd_hbm_share"],
                 100 * r["b_bwd_hbm_share"], r["c_fwd_ms"], r["c_bwd_ms"], r["d_fwd_ms"], r["d_bwd_ms"],
                 r["h2d_target_bytes_onehot_u8"] / 1e6, r["h2d_target_bytes_label_u8"] / 1e6))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
