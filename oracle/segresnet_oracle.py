"""CPU restatement of ``monai.networks.nets.SegResNet`` (Myronenko's BraTS 2018 network, which the reference builds by name
through the ``from monai.networks.nets import *`` in unet3d/models/pytorch/__init__.py:1) for the configuration subset the GPU
path implements.  TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

PARITY UNPINNED: MONAI is a third-party dependency that is not vendored under /root/reference and is not installed in this
image.  The network below is restated from MONAI's public source (monai/networks/nets/segresnet.py and
monai/networks/blocks/segresnet_block.py), with its defaults spatial_dims=3, init_filters=8, in_channels=1, out_channels=2,
dropout_prob=None, act=("RELU", {"inplace": True}), norm=("GROUP", {"num_groups": 8}), use_conv_final=True,
blocks_down=(1, 2, 2, 4), blocks_up=(1, 1, 1), upsample_mode="nontrainable":

  conv(ci, co, k=3, s=1, bias=False)  Conv3d with padding k // 2;  F = init_filters, L = len(blocks_down)
  ResBlock(C)                         y = conv2(act(norm2(conv1(act(norm1(x)))))) + x, GroupNorm(num_groups, C) affine eps 1e-5,
                                      C -> C 3x3x3 bias-free convs
  forward                             x = convInit(x) [-> Dropout3d(dropout_prob): per (n, c), scaled by 1 / (1 - p)]
                                      level i: x = pre_conv_i(x) (Identity at i = 0, else conv(F 2^(i-1), F 2^i, 3, stride 2) on
                                      the raw level output), then blocks_down[i] x ResBlock(F 2^i); down_x[i] = x
                                      up stage i = 0..L-2, C = F 2^(L-2-i): x = upsample2x(conv1x1(2C -> C)(x)) + down_x[L-2-i]
                                      (trilinear, align_corners=False), then blocks_up[i] x ResBlock(C)
                                      head: conv_final = GroupNorm(F) -> act -> conv(F, out_channels, 1, bias=True)
  state dict                          convInit.conv.weight; down_layers.{i}.0.conv.weight (i > 0) then the ResBlocks
                                      down_layers.{i}.{1..blocks_down[i]}.*; up_layers.{i}.{0..}.* (all of up_layers before
                                      up_samples); up_samples.{i}.0.conv.weight [C, 2C, 1, 1, 1]; conv_final.0.weight / .bias,
                                      conv_final.2.conv.weight / .bias.  A ResBlock's own order: norm1.weight, norm1.bias,
                                      norm2.weight, norm2.bias, conv1.conv.weight, conv2.conv.weight.
  init                                PyTorch's defaults (no custom init).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F


def segresnet_state_dict_spec(in_channels: int = 1, out_channels: int = 2, init_filters: int = 8,
                              blocks_down: Sequence[int] = (1, 2, 2, 4), blocks_up: Sequence[int] = (1, 1, 1)
                              ) -> List[Tuple[str, Tuple[int, ...]]]:
    """Ordered (key, shape) list in MONAI's module registration order."""
    L, f = len(blocks_down), init_filters
    spec: List[Tuple[str, Tuple[int, ...]]] = [("convInit.conv.weight", (f, in_channels, 3, 3, 3))]

    def block(prefix, c):
        for n in ("norm1", "norm2"):
            spec.append((f"{prefix}.{n}.weight", (c,)))
            spec.append((f"{prefix}.{n}.bias", (c,)))
        spec.append((f"{prefix}.conv1.conv.weight", (c, c, 3, 3, 3)))
        spec.append((f"{prefix}.conv2.conv.weight", (c, c, 3, 3, 3)))
    for i, nb in enumerate(blocks_down):
        if i > 0:
            spec.append((f"down_layers.{i}.0.conv.weight", (f << i, f << (i - 1), 3, 3, 3)))
        for b in range(1, nb + 1):
            block(f"down_layers.{i}.{b}", f << i)
    for i, nb in enumerate(blocks_up):
        for b in range(nb):
            block(f"up_layers.{i}.{b}", f << (L - 2 - i))
    for i in range(L - 1):
        c = f << (L - 2 - i)
        spec.append((f"up_samples.{i}.0.conv.weight", (c, 2 * c, 1, 1, 1)))
    spec += [("conv_final.0.weight", (f,)), ("conv_final.0.bias", (f,)),
             ("conv_final.2.conv.weight", (out_channels, f, 1, 1, 1)), ("conv_final.2.conv.bias", (out_channels,))]
    return spec


def make_segresnet_state_dict(in_channels: int = 1, out_channels: int = 2, init_filters: int = 8, blocks_down=(1, 2, 2, 4),
                              blocks_up=(1, 1, 1), seed: int = 0, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """seeded state dict: He-scaled conv weights (the residual sums stay O(1) through the depth), norm gains 1 + 0.2 N(0, 1),
    biases 0.1 N(0, 1)"""
    out = {}
    for idx, (key, shape) in enumerate(segresnet_state_dict_spec(in_channels, out_channels, init_filters, blocks_down, blocks_up)):
        g = torch.Generator().manual_seed(9000011 * (seed + 1) + idx)
        if len(shape) == 1 and key.endswith("weight"):
            t = 1.0 + 0.2 * torch.randn(shape, generator=g, dtype=torch.float64)
        elif key.endswith(".bias"):
            t = 0.1 * torch.randn(shape, generator=g, dtype=torch.float64)
        else:
            fan_in = shape[1] * shape[2] * shape[3] * shape[4]
            t = torch.randn(shape, generator=g, dtype=torch.float64) * (2.0 / fan_in) ** 0.5
        out[key] = t.to(dtype)
    return out


def _act(x, slope):
    return F.leaky_relu(x, slope) if slope else F.relu(x)


def _res_block(sd, prefix, x, groups, slope):
    y = _act(F.group_norm(x, groups, sd[f"{prefix}.norm1.weight"], sd[f"{prefix}.norm1.bias"], eps=1e-5), slope)
    y = F.conv3d(y, sd[f"{prefix}.conv1.conv.weight"], None, padding=1)
    y = _act(F.group_norm(y, groups, sd[f"{prefix}.norm2.weight"], sd[f"{prefix}.norm2.bias"], eps=1e-5), slope)
    y = F.conv3d(y, sd[f"{prefix}.conv2.conv.weight"], None, padding=1)
    return y + x


def segresnet_forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, blocks_down=(1, 2, 2, 4), blocks_up=(1, 1, 1),
                      num_groups: int = 8, dropout_scale: Optional[torch.Tensor] = None, slope: float = 0.0) -> torch.Tensor:
    """Functional forward.  dropout_scale: (N, init_filters) Dropout3d channel scale applied to convInit's output (None = eval);
    slope: the activation's negative slope (0 = ReLU)."""
    L = len(blocks_down)
    x = F.conv3d(x, sd["convInit.conv.weight"], None, padding=1)
    if dropout_scale is not None:
        x = x * dropout_scale.to(x.dtype)[:, :, None, None, None]
    down_x = []
    for i, nb in enumerate(blocks_down):
        if i > 0:
            x = F.conv3d(x, sd[f"down_layers.{i}.0.conv.weight"], None, stride=2, padding=1)
        for b in range(1, nb + 1):
            x = _res_block(sd, f"down_layers.{i}.{b}", x, num_groups, slope)
        down_x.append(x)
    for i, nb in enumerate(blocks_up):
        x = F.conv3d(x, sd[f"up_samples.{i}.0.conv.weight"], None)
        x = F.interpolate(x, scale_factor=2, mode="trilinear", align_corners=False) + down_x[L - 2 - i]
        for b in range(nb):
            x = _res_block(sd, f"up_layers.{i}.{b}", x, num_groups, slope)
    x = _act(F.group_norm(x, num_groups, sd["conv_final.0.weight"], sd["conv_final.0.bias"], eps=1e-5), slope)
    return F.conv3d(x, sd["conv_final.2.conv.weight"], sd["conv_final.2.conv.bias"])
