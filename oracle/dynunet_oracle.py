"""CPU restatement of ``monai.networks.nets.DynUNet`` (the model the reference's example configs train:
examples/brats2020/brats2020_config.json:2-107) for the configuration subset the GPU path implements.
TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

PARITY UNPINNED: MONAI is a third-party dependency that is not vendored under /root/reference and is not installed in this
image (requirements.txt:4 leaves it unpinned; Dockerfile:1 uses ``projectmonai/monai:latest``).  The block semantics
below are restated from MONAI's public source (monai/networks/nets/dynunet.py and monai/networks/blocks/dynunet_block.py):

  UnetBasicBlock(in, out, k, s):  conv(k, stride s, pad k//2, bias-free) -> InstanceNorm3d(affine, eps 1e-5) -> LeakyReLU(0.01)
                                  -> conv(k, stride 1) -> InstanceNorm3d -> LeakyReLU
  UnetUpBlock(in, out):           ConvTranspose3d(in, out, kernel = stride = upsample_kernel_size, bias=trans_bias)
                                  -> cat((up, skip), 1) -> UnetBasicBlock(2 out, out, k, 1)
  UnetOutBlock(in, out):          1x1x1 conv with bias
  DynUNet.forward:                input_block -> downsamples[...] -> bottleneck, then upsamples[i](x, skip) mirrored, output_block
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import torch
import torch.nn.functional as F


def dynunet_state_dict_spec(in_channels: int, out_channels: int, filters: Sequence[int]) -> List[Tuple[str, Tuple[int, ...]]]:
    """Ordered (key, shape) list in MONAI's module registration order (skip_layers.* aliases omitted)."""
    L = len(filters)
    spec: List[Tuple[str, Tuple[int, ...]]] = []

    def block(prefix, cin, cout):
        spec.append((f"{prefix}.conv1.conv.weight", (cout, cin, 3, 3, 3)))
        spec.append((f"{prefix}.conv2.conv.weight", (cout, cout, 3, 3, 3)))
        for n in ("norm1", "norm2"):
            spec.append((f"{prefix}.{n}.weight", (cout,)))
            spec.append((f"{prefix}.{n}.bias", (cout,)))
    for i in range(L):
        name = "input_block" if i == 0 else "bottleneck" if i == L - 1 else f"downsamples.{i - 1}"
        block(name, in_channels if i == 0 else filters[i - 1], filters[i])
    for u in range(L - 1):
        lo, hi = L - 1 - u, L - 2 - u
        spec.append((f"upsamples.{u}.transp_conv.conv.weight", (filters[lo], filters[hi], 2, 2, 2)))
        block(f"upsamples.{u}.conv_block", 2 * filters[hi], filters[hi])
    spec.append(("output_block.conv.conv.weight", (out_channels, filters[0], 1, 1, 1)))
    spec.append(("output_block.conv.conv.bias", (out_channels,)))
    return spec


def make_dynunet_state_dict(in_channels, out_channels, filters, seed=0, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    out = {}
    for idx, (key, shape) in enumerate(dynunet_state_dict_spec(in_channels, out_channels, filters)):
        g = torch.Generator().manual_seed(7000003 * (seed + 1) + idx)
        if ".norm" in key and key.endswith("weight"):
            t = 1.0 + 0.2 * torch.randn(shape, generator=g, dtype=torch.float64)
        elif key.endswith(".bias"):
            t = 0.1 * torch.randn(shape, generator=g, dtype=torch.float64)
        else:
            fan_in = shape[1] * shape[2] * shape[3] * shape[4]
            t = torch.randn(shape, generator=g, dtype=torch.float64) * (2.0 / fan_in) ** 0.5
        out[key] = t.to(dtype)
    return out


def _basic_block(sd, prefix, x, stride, slope):
    x = F.conv3d(x, sd[f"{prefix}.conv1.conv.weight"], None, stride=stride, padding=1)
    x = F.leaky_relu(F.instance_norm(x, weight=sd[f"{prefix}.norm1.weight"], bias=sd[f"{prefix}.norm1.bias"], eps=1e-5), slope)
    x = F.conv3d(x, sd[f"{prefix}.conv2.conv.weight"], None, stride=1, padding=1)
    return F.leaky_relu(F.instance_norm(x, weight=sd[f"{prefix}.norm2.weight"], bias=sd[f"{prefix}.norm2.bias"], eps=1e-5), slope)


def dynunet_forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, n_levels: int, slope: float = 0.01) -> torch.Tensor:
    L = n_levels
    skips = []
    for i in range(L):
        name = "input_block" if i == 0 else "bottleneck" if i == L - 1 else f"downsamples.{i - 1}"
        x = _basic_block(sd, name, x, 1 if i == 0 else 2, slope)
        if i < L - 1:
            skips.append(x)
    for u in range(L - 1):
        x = F.conv_transpose3d(x, sd[f"upsamples.{u}.transp_conv.conv.weight"], None, stride=2)
        x = torch.cat((x, skips[L - 2 - u]), dim=1)
        x = _basic_block(sd, f"upsamples.{u}.conv_block", x, 1, slope)
    return F.conv3d(x, sd["output_block.conv.conv.weight"], sd["output_block.conv.conv.bias"])
