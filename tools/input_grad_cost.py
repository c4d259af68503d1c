"""Cost of the input gradient at the C2 size (UNet3D, 2 x 4 x 128^3, base_width 32, bf16): b200unet_plan_input_grad timed with CUDA
events next to b200unet_plan_backward on the same plan and workspace.  Both calls only read the workspace the forward left
and overwrite their outputs, so they can be repeated.  Prints the card name and power limit beside the numbers.

    python tools/input_grad_cost.py [--reps 20] [--precision bf16|split]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("3dunetcnn_b200")
models = pkg.models


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:  # noqa: BLE001
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--precision", default="bf16")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    torch.manual_seed(0)
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=32, precision=args.precision).cuda()
    model.train()
    x = torch.randn(2, 4, 128, 128, 128, device="cuda", requires_grad=True)
    t = (torch.rand(2, 3, 128, 128, 128, device="cuda") > 0.7).to(torch.uint8)
    crit = pkg.DiceLoss(sigmoid=True)
    for _ in range(2):                                    # warm-up through the module (flagged plan, full backward + input gradient)
        model.zero_grad(set_to_none=True)
        x.grad = None
        crit(model(x), t).backward()
    torch.cuda.synchronize()
    plan = model._plan_for(x, inference_only=False, input_grad=True)
    params = model.ordered_parameters()
    grads = [torch.empty_like(p) for p in params]
    dlogits = torch.randn(2, 3, 128, 128, 128, device="cuda") * 1e-6
    dx = torch.empty_like(x)
    ws, st = plan.workspace.data_ptr(), pkg.lib.stream_ptr()
    pa, ga = models._ptr_array(params), models._ptr_array(grads)

    def bwd():
        pkg.lib.check(plan.lib.b200unet_plan_backward(plan.handle, dlogits.data_ptr(), pa, ga, ws, st), "plan_backward")

    def igrad():
        pkg.lib.check(plan.lib.b200unet_plan_input_grad(plan.handle, dx.data_ptr(), ws, st), "plan_input_grad")

    res = {}
    for name, fn in (("backward", bwd), ("input_grad", igrad)):
        fn()
        torch.cuda.synchronize()
        launches = plan.last_launches()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(args.reps):
            fn()
        ev[1].record()
        torch.cuda.synchronize()
        res[name] = dict(ms=ev[0].elapsed_time(ev[1]) / args.reps, launches=launches)
    S = 128 ** 3
    cp, C0, nf = 8, 32, 4
    elt = 4 if args.precision == "split" else 2                   # bytes per stored element (hi [+ lo])
    # algorithmic bytes: sample dgrad reads dOut (C0) and writes 8 channels; the fused kernel reads dz, x, r (8 channels) and writes fp32
    bytes_sample = 2 * S * (C0 + cp) * elt
    bytes_fused = 2 * S * (3 * cp * elt + nf * 4)
    res["input_grad"]["algorithmic_bytes"] = bytes_sample + bytes_fused
    res["input_grad"]["GB_per_s"] = (bytes_sample + bytes_fused) / (res["input_grad"]["ms"] * 1e-3) / 1e9
    out = dict(device=torch.cuda.get_device_name(), power_limit=power_limit(), precision=args.precision, shape=[2, 4, 128, 128, 128],
               base_width=32, reps=args.reps, **res, input_grad_over_backward=res["input_grad"]["ms"] / res["backward"]["ms"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
