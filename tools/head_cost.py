"""Cost of the 1x1x1 head by class count at the C2 size (2 x 128^3 voxels, 32 channels into the head, bf16).

For each n_out: b200unet_head_fwd and b200unet_head_bwd timed with CUDA events over many launches after warm-up, the HBM
bytes each direction needs (computed from shapes: x, logits / dlogits, dx), the achieved GB/s and its share of the H100
SXM data-sheet 3.35 TB/s, and DiceLoss(sigmoid=True) forward + backward for context.  Then a full UNet3D training step
(forward + Dice + backward, eager, no optimizer) at 3 and 104 outputs in volumes/s.  n_out 3 and 8 run the SIMT head, the
others the tensor-core head.  Prints the card name and power limit of the same run.

    python tools/head_cost.py [--reps 50] [--steps 5] [--out FILE.json]
"""
import argparse
import ctypes as C
import importlib
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("3dunetcnn_b200")
L = pkg.lib

HBM_PEAK = 3.35e12
N, S, CH = 2, 128, 32


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:  # noqa: BLE001
        return "unknown"


def time_ms(fn, reps, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def head_row(n_out, reps):
    lib = L.load_library()
    dev = "cuda"
    vox = N * S ** 3
    g = torch.Generator(device=dev).manual_seed(0)
    x = L.Act(torch.randn(N, S, S, S, CH, device=dev, generator=g).to(torch.bfloat16))
    dx = L.Act.empty(N, S, S, S, CH)
    w = torch.randn(n_out, CH, device=dev, generator=g) / CH ** 0.5
    dw = torch.empty_like(w)
    logits = torch.empty(N, n_out, S, S, S, device=dev)
    dlogits = torch.randn(N, n_out, S, S, S, device=dev, generator=g)
    scratch = torch.empty(int(lib.b200unet_head_bwd_scratch_bytes(n_out, CH)), dtype=torch.uint8, device=dev)
    xc, dxc = x.ct(), dx.ct()

    def fwd():
        L.check(lib.b200unet_head_fwd(C.byref(xc), w.data_ptr(), n_out, 0, logits.data_ptr(), L.stream_ptr()), "head_fwd")

    def bwd():
        L.check(lib.b200unet_head_bwd(C.byref(xc), w.data_ptr(), n_out, dlogits.data_ptr(), C.byref(dxc), dw.data_ptr(),
                                      scratch.data_ptr(), L.stream_ptr()), "head_bwd")

    t_fwd, t_bwd = time_ms(fwd, reps), time_ms(bwd, reps)
    b_fwd = vox * (CH * 2 + n_out * 4)                 # read x, write logits
    b_bwd = vox * (CH * 2 + n_out * 4 + CH * 2)        # read x and dlogits, write dx
    target = (torch.rand(N, n_out, S, S, S, device=dev, generator=g) > 0.7).to(torch.uint8)
    crit = pkg.DiceLoss(sigmoid=True)
    lg = logits.detach().requires_grad_(True)

    def dice():
        lg.grad = None
        crit(lg, target).backward()
    t_dice = time_ms(dice, max(reps // 5, 5))
    del logits, dlogits, target, lg
    row = dict(n_out=n_out, head="simt" if n_out <= 8 else "tensor-core", fwd_ms=t_fwd, bwd_ms=t_bwd, fwd_bytes=b_fwd, bwd_bytes=b_bwd,
               fwd_GBps=b_fwd / t_fwd / 1e6, bwd_GBps=b_bwd / t_bwd / 1e6, fwd_hbm_frac=b_fwd / t_fwd / 1e-3 / HBM_PEAK,
               bwd_hbm_frac=b_bwd / t_bwd / 1e-3 / HBM_PEAK, dice_fwd_bwd_ms=t_dice)
    torch.cuda.empty_cache()
    return row


def step_rate(n_out, steps):
    dev = "cuda"
    model = pkg.UNet3D(precision="bf16", n_features=4, n_outputs=n_out, base_width=32).to(dev)
    model.train()
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(N, 4, S, S, S, device=dev, generator=g)
    t = (torch.rand(N, n_out, S, S, S, device=dev, generator=g) > 0.7).to(torch.uint8)
    crit = pkg.DiceLoss(sigmoid=True)

    def step():
        model.zero_grad(set_to_none=True)
        crit(model(x), t).backward()
    ms = time_ms(step, steps, warmup=3)
    del model
    torch.cuda.empty_cache()
    return dict(n_out=n_out, step_ms=ms, volumes_per_s=N / ms * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("head_cost.py needs a CUDA device")
    card = dict(name=torch.cuda.get_device_name(), power_limit=power_limit())
    print("card: %s, power limit %s" % (card["name"], card["power_limit"]))
    rows = []
    print("%6s %-11s %9s %9s %9s %9s %7s %7s %10s" % ("n_out", "head", "fwd ms", "fwd GB/s", "bwd ms", "bwd GB/s", "fwd %", "bwd %",
                                                    "dice ms"))
    for n_out in (3, 8, 9, 16, 32, 64, 104, 128):
        r = head_row(n_out, args.reps)
        rows.append(r)
        print("%6d %-11s %9.3f %9.0f %9.3f %9.0f %6.1f%% %6.1f%% %10.3f" % (r["n_out"], r["head"], r["fwd_ms"], r["fwd_GBps"], r["bwd_ms"],
                                                                          r["bwd_GBps"], 100 * r["fwd_hbm_frac"], 100 * r["bwd_hbm_frac"],
                                                                          r["dice_fwd_bwd_ms"]))
    steps = [step_rate(n, args.steps) for n in (3, 104)]
    for s in steps:
        print("UNet3D C2-size training step (eager forward + Dice + backward), %3d outputs: %.2f ms, %.2f volumes/s"
              % (s["n_out"], s["step_ms"], s["volumes_per_s"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=card, heads=rows, steps=steps), f, indent=1)


if __name__ == "__main__":
    main()
