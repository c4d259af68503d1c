"""Generate tests/golden/input_grad.npz: the gradient of the Dice loss with respect to the network INPUT, from the UNMODIFIED
reference UNet3D in fp64 on CPU (train mode, the shared Dropout3d mask), exactly as make_golden.py runs it.

Run in the build container (needs /root/reference):   python tests/golden/make_golden_input_grad.py
Inputs and weights are not stored: they are regenerated from the seeds of recipe.py.  Per case: the norm of x.grad, its
per-(n, c) norms and a stride-4 spatial subsample.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import UNetConfig, make_state_dict, dice_loss  # noqa: E402
from oracle.ref_loader import reference_unet3d  # noqa: E402

sys.path.insert(0, HERE)
from recipe import CASES, golden_inputs, dropout_mask  # noqa: E402

# every recipe case, plus the identity residual branch of the first block (n_features == base_width: no `sample` conv)
INPUT_GRAD_CASES = dict(CASES)
INPUT_GRAD_CASES["identity_bw8_n8_32"] = (dict(n_features=8, n_outputs=3, base_width=8), (1, 8, 32, 32, 32))
SUB = (slice(None), slice(None), slice(None, None, 4), slice(None, None, 4), slice(None, None, 4))


def run_case(kw, shape):
    cfg = UNetConfig(**kw)
    model = reference_unet3d(**kw).double()
    model.load_state_dict(make_state_dict(cfg, seed=0, dtype=torch.float64), strict=True)
    x, t, g3 = golden_inputs(shape, cfg.n_outputs)
    x = x.double().requires_grad_(True)
    mask = dropout_mask(shape[0], cfg.enc_widths()[0], cfg.dropout, g3)
    model.encoder.layers[0].dropout.forward = lambda inp: inp * mask.to(inp.dtype).view(inp.shape[0], inp.shape[1], 1, 1, 1)
    model.train()
    loss = dice_loss(model(x), t)
    loss.backward()
    return x.grad.detach()


def main():
    out = {}
    for name, (kw, shape) in INPUT_GRAD_CASES.items():
        dx = run_case(kw, shape)
        out[name + "::norm"] = np.float64(dx.norm())
        out[name + "::nc_norms"] = dx.flatten(2).norm(dim=2).numpy()
        out[name + "::sub4"] = dx[SUB].numpy().astype(np.float32)
        print(name, "|dx|", float(dx.norm()))
    path = os.path.join(HERE, "input_grad.npz")
    np.savez_compressed(path, **out)
    print("->", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
