"""The bar to meet: the reference model's op graph (oracle's functional restatement == the reference's nn.Module
graph) executed by torch/cuDNN on the same GPU: fp32 (TF32 off), and bf16 autocast (+channels_last_3d).
Prints one JSON line per variant.  Not part of the product path."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import UNetConfig, make_state_dict, unet3d_forward, dice_loss  # noqa: E402

cfg = UNetConfig(n_features=4, n_outputs=3, base_width=32)
dev = "cuda"
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
x = torch.randn(2, 4, 128, 128, 128, device=dev)
t = (torch.rand(2, 3, 128, 128, 128, device=dev) > 0.7).to(torch.uint8)


def run(name, autocast, channels_last, benchmark):
    torch.backends.cudnn.benchmark = benchmark
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = {k: v.to(dev).requires_grad_(True) for k, v in make_state_dict(cfg, seed=0).items()}
    xx = x.contiguous(memory_format=torch.channels_last_3d) if channels_last else x
    if channels_last:
        sd = {k: (v.detach().contiguous(memory_format=torch.channels_last_3d).requires_grad_(True) if v.dim() == 5 else v) for k, v in sd.items()}

    def step():
        for p in sd.values():
            p.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            out = unet3d_forward(sd, xx, cfg)
        loss = dice_loss(out.float(), t)
        loss.backward()
        return loss
    try:
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            loss = step()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        print(json.dumps({"variant": name, "ms_per_step": ms, "volumes_per_s": 2 / (ms / 1e3), "loss": float(loss),
                          "mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30}), flush=True)
    except Exception as e:  # noqa
        print(json.dumps({"variant": name, "error": repr(e)[:300]}), flush=True)
    torch.cuda.empty_cache()


run("cudnn bf16 autocast, NCDHW, benchmark off", True, False, False)
run("cudnn bf16 autocast, NCDHW, benchmark on", True, False, True)
run("cudnn bf16 autocast, channels_last_3d, benchmark on", True, True, True)
run("cudnn fp32 (TF32 off), NCDHW, benchmark on", False, False, True)
