"""Cost of resampling a prediction onto its image file's grid (``prepost.resample_to_match``, the step
``volumetric_predictions(resample=True)`` adds per item).

Cases (tests/resample_cases.py builds the grids: orientation, foreground crop and resize, as the dataset applies them):
  BraTS  3 channels, 128^3 prediction -> 240 x 240 x 155 file grid (LPS file oriented to RAS)
  SPPIN  1 channel, 192^3 prediction -> 256 x 256 x 160 anisotropic file grid under an oblique, non-diagonal affine, axes permuted
Timed with CUDA events after warm-up, medians of --reps:
  call    prepost.resample_to_match (index map composed on the host in fp64, one kernel)
  kernel  b200unet_resample_to_grid alone
  torch   a torch GPU restatement: affine_grid + grid_sample (bilinear, border, align_corners=False) in fp32
  host    the path it replaces: device-to-host copy of the prediction, then torch CPU affine_grid + grid_sample in fp64 (host
          clock, --host-reps, torch's default CPU threads unless --host-threads is given)
Compulsory bytes: the prediction read once and the resampled volume written once, fp32; the table gives the call's and the
kernel's share of the H100 SXM data-sheet 3.35 TB/s on them.  Prints the card name and power limit of the same run.

    python tools/resample_cost.py [--reps 50] [--out FILE.json]
"""
import argparse
import ctypes as C
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
pkg = importlib.import_module("3dunetcnn_b200")
import resample_cases as rc  # noqa: E402

HBM_PEAK = 3.35e12
CASES = {"BraTS": ("brats", 3), "SPPIN": ("sppin", 1)}


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


def torch_restatement(x, m, dst_shape):
    """x [C, D, H, W] resampled through the 3x4 index map m with torch ops, in x's dtype and on x's device"""
    src = torch.tensor(x.shape[1:], dtype=torch.float64)
    dst = torch.tensor(dst_shape, dtype=torch.float64)
    # normalised target u -> target index ((u + 1) dst - 1) / 2 -> source index m p -> normalised source (2 q + 1) / src - 1
    to_idx = torch.eye(4, dtype=torch.float64)
    to_idx[:3, :3] = torch.diag(dst / 2)
    to_idx[:3, 3] = (dst - 1) / 2
    to_norm = torch.eye(4, dtype=torch.float64)
    to_norm[:3, :3] = torch.diag(2 / src)
    to_norm[:3, 3] = 1 / src - 1
    mm = torch.eye(4, dtype=torch.float64)
    mm[:3] = torch.from_numpy(m)
    theta = (to_norm @ mm @ to_idx)[:3]
    perm = [2, 1, 0]                                                      # (d, h, w) -> grid's (x, y, z) = (w, h, d)
    theta = theta[perm][:, perm + [3]].to(x.dtype).to(x.device)
    grid = F.affine_grid(theta[None], [1, x.shape[0]] + list(dst_shape), align_corners=False)
    return F.grid_sample(x[None], grid, mode="bilinear", padding_mode="border", align_corners=False)[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--host-threads", type=int, default=0, help="torch CPU threads of the host path (0: torch's default)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "resample_cost needs a CUDA device"
    if args.host_threads:
        torch.set_num_threads(args.host_threads)
    dev = torch.device("cuda")
    lib = pkg.lib.load_library()
    rows = []
    for name, (grid, c) in CASES.items():
        a0, shape, a, pshape = rc.grid(grid)
        x = torch.rand((c,) + pshape, generator=torch.Generator().manual_seed(0)).to(dev)
        m = pkg.prepost.index_map(a, a0)
        out = torch.empty((c,) + shape, dtype=torch.float32, device=dev)
        mc = (C.c_double * 12)(*m.ravel().tolist())

        def kernel():
            pkg.lib.check(lib.b200unet_resample_to_grid(x.data_ptr(), c, *pshape, mc, 0, out.data_ptr(), *shape, pkg.lib.stream_ptr()))
        call = timed(lambda: pkg.prepost.resample_to_match(x, a, a0, shape), args.reps)
        kern = timed(kernel, args.reps)
        ref = timed(lambda: torch_restatement(x, m, shape), args.reps)
        y = pkg.prepost.resample_to_match(x, a, a0, shape)
        diff_torch = float((y - torch_restatement(x, m, shape)).abs().max())
        ts = []
        for _ in range(args.host_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            yh = torch_restatement(x.cpu().double(), m, shape)
            ts.append((time.perf_counter() - t0) * 1e3)
        host = statistics.median(ts)
        diff_host = float((y.cpu().double() - yh).abs().max())
        byt = 4 * c * (int(np.prod(pshape)) + int(np.prod(shape)))
        rows.append({"case": name, "channels": c, "prediction": list(pshape), "file": list(shape), "call_ms": call, "kernel_ms": kern,
                     "torch_gpu_ms": ref, "host_ms": host, "host_threads": torch.get_num_threads(), "bytes": byt,
                     "call_share_of_hbm": byt / (call * 1e-3) / HBM_PEAK, "kernel_share_of_hbm": byt / (kern * 1e-3) / HBM_PEAK,
                     "max_abs_vs_torch_gpu": diff_torch, "max_abs_vs_host_fp64": diff_host})
    info = {"device": torch.cuda.get_device_name(), "power_limit": power_limit(), "reps": args.reps, "rows": rows}
    print("%s, power limit %s, medians of %d" % (info["device"], info["power_limit"], args.reps))
    print("| case | MB moved | call ms | share of HBM | kernel ms | share of HBM | torch GPU ms | host (D2H + CPU fp64) ms, %d threads |"
          % rows[0]["host_threads"])
    for r in rows:
        print("| %s | %.0f | %.3f | %.0f %% | %.3f | %.0f %% | %.3f | %.0f |" % (
            r["case"], r["bytes"] / 1e6, r["call_ms"], 100 * r["call_share_of_hbm"], r["kernel_ms"], 100 * r["kernel_share_of_hbm"],
            r["torch_gpu_ms"], r["host_ms"]))
    for r in rows:
        print("%s: max abs vs torch GPU fp32 %.2e, vs host fp64 %.2e" % (r["case"], r["max_abs_vs_torch_gpu"], r["max_abs_vs_host_fp64"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
