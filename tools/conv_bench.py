"""Per-layer micro-benchmark of the convolution kernels at the C2 layer shapes (batch 2): TFLOP/s per layer for
forward (mode 0 + stats), the wgrad kernel, and the halo-mode data gradients of the C2 step (dgrad: mode 1); B200UNET_NO_HALO=1 keeps
every convolution on the per-tap kernel (A/B).  Usage: python tools/conv_bench.py [fwd|epi|wgrad|dgrad|all] [reps]"""
import importlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dunetcnn_b200")
L = pkg.lib
DEV = "cuda"
SHAPES = [(8, 32, 128), (32, 32, 128), (64, 32, 128), (32, 64, 64), (64, 64, 64), (128, 128, 64), (64, 128, 32),
          (128, 128, 32), (256, 256, 32), (128, 256, 16), (256, 256, 16)]
# how many times each shape occurs in one C2 forward (for the weighted total)
COUNT = {(8, 32, 128): 1, (32, 32, 128): 2, (64, 32, 128): 1, (32, 64, 64): 1, (64, 64, 64): 3, (128, 128, 64): 2,
         (64, 128, 32): 1, (128, 128, 32): 3, (256, 256, 32): 2, (128, 256, 16): 1, (256, 256, 16): 9}
# the mode-1 data gradients (GroupNorm/ReLU backward epilogue) of the C2 step at 128^3 that run in halo mode: (Cin, Cout, r) of
# the data-gradient convolution, and how many times each occurs in one C2 backward
DGRAD = {(32, 32, 128): 2, (32, 64, 128): 1, (32, 8, 128): 1}


def timeit(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    tag = {k: os.environ.get(k) for k in ("B200UNET_NO_HALO",) if os.environ.get(k)}
    tot_ms = {"fwd": 0.0, "wgrad": 0.0}
    tot_flop = 0.0
    for (ci, co, r) in SHAPES:
        n = 2
        x = L.Act.empty(n, r, r, r, ci)
        x.hi.normal_()
        w = torch.randn(co, ci, 3, 3, 3, device=DEV) / (ci * 27) ** 0.5
        whi, wlo, cop, cip, _ = L.pack_weights(w, 0)
        y = L.Act.empty(n, r, r, r, co)
        stats = torch.zeros(n, co, 2, dtype=torch.float64, device=DEV)
        flop = 2.0 * n * r ** 3 * ci * co * 27
        out = {"ci": ci, "co": co, "r": r}
        if what in ("fwd", "all"):
            ms = timeit(lambda: L.conv3d(x, whi, wlo, 3, 1, y, cop, cip, stats=stats, stats_ld=co), reps)
            out["fwd_ms"] = round(ms, 4)
            out["fwd_tflops"] = round(flop / ms / 1e9, 1)
            tot_ms["fwd"] += ms * COUNT[(ci, co, r)]
        if what in ("epi", "all"):
            res = L.Act.empty(n, r, r, r, co)
            res.hi.normal_()
            ms = timeit(lambda: L.conv3d(x, whi, wlo, 3, 1, y, cop, cip, res=res, stats=stats, stats_ld=co), reps)
            out["res_ms"] = round(ms, 4)
            out["res_tflops"] = round(flop / ms / 1e9, 1)
            tot_ms.setdefault("res", 0.0)
            tot_ms["res"] += ms * COUNT[(ci, co, r)]
            coef = torch.rand(n, co, 4, device=DEV)
            bst = torch.zeros(n, co, 2, dtype=torch.float64, device=DEV)
            ms = timeit(lambda: L.conv3d(x, whi, wlo, 3, 1, y, cop, cip, mode=1, gn_x=res, coef=coef, coef_ld=co, bstats=bst), reps)
            out["mode1_ms"] = round(ms, 4)
            out["mode1_tflops"] = round(flop / ms / 1e9, 1)
            tot_ms.setdefault("mode1", 0.0)
            tot_ms["mode1"] += ms * COUNT[(ci, co, r)]
        if what in ("wgrad", "all"):
            dy = L.Act.empty(n, r, r, r, co)
            dy.hi.normal_()
            dw = torch.zeros(27, cip, cop, device=DEV)
            ms = timeit(lambda: L.conv3d_wgrad(x, dy, 3, 1, cip, cop, dw), reps)
            out["wgrad_ms"] = round(ms, 4)
            out["wgrad_tflops"] = round(flop / ms / 1e9, 1)
            tot_ms["wgrad"] += ms * COUNT[(ci, co, r)]
        tot_flop += flop * COUNT[(ci, co, r)]
        print("[convbench]", json.dumps({**tag, **out}), flush=True)
    if what in ("dgrad", "all"):
        tot_ms["dgrad"], dflop = 0.0, 0.0
        for (ci, co, r), cnt in DGRAD.items():
            n = 2
            dy = L.Act.empty(n, r, r, r, ci)
            dy.hi.normal_()
            w = torch.randn(co, ci, 3, 3, 3, device=DEV) / (ci * 27) ** 0.5
            whi, wlo, cop, cip, _ = L.pack_weights(w, 0)
            gx = L.Act.empty(n, r, r, r, co)
            gx.hi.normal_()
            dz = L.Act.empty(n, r, r, r, co)
            coef = torch.rand(n, co, 4, device=DEV)
            bst = torch.zeros(n, co, 2, dtype=torch.float64, device=DEV)
            route = L.conv3d_route(dy, whi, wlo, 3, 1, dz, cop, cip, mode=1, gn_x=gx, coef=coef, coef_ld=co, bstats=bst)
            ms = timeit(lambda: L.conv3d(dy, whi, wlo, 3, 1, dz, cop, cip, mode=1, gn_x=gx, coef=coef, coef_ld=co, bstats=bst), reps)
            flop = 2.0 * n * r ** 3 * ci * co * 27
            print("[convbench]", json.dumps({**tag, "dgrad_ci": ci, "co": co, "r": r, "route": [route["kind"], route["bn"], route["kc"]],
                                             "grid": route["grid"], "mode1_ms": round(ms, 4), "mode1_tflops": round(flop / ms / 1e9, 1)}),
                  flush=True)
            tot_ms["dgrad"] += ms * cnt
            dflop += flop * cnt
        v = tot_ms.pop("dgrad")
        print("[convbench] dgrad weighted total: %.3f ms per C2 backward -> %.1f TFLOP/s  %s" % (v, dflop / v / 1e9, tag), flush=True)
    for k, v in tot_ms.items():
        if v:
            print("[convbench] %s weighted total: %.3f ms per C2 pass -> %.1f TFLOP/s  %s" % (k, v, tot_flop / v / 1e9, tag), flush=True)


if __name__ == "__main__":
    main()
