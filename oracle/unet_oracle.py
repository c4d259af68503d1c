"""CPU restatement of ``monai.networks.nets.UNet`` (the network of MONAI's 3D tutorials, which the reference builds by name
through the ``from monai.networks.nets import *`` in unet3d/models/pytorch/__init__.py:1) for the configuration subset the GPU
path implements.  TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

PARITY UNPINNED: MONAI is a third-party dependency that is not installed in this image.  The network below is restated from
MONAI's public source (monai/networks/nets/unet.py, monai/networks/blocks/convolutions.py ``Convolution`` / ``ResidualUnit``,
monai/networks/layers/simplelayers.py ``SkipConnection``) with kernel_size = up_kernel_size = 3, every stride 2, dropout 0 and
adn_ordering "NDA":

  Convolution(ci, co, s)     conv k3 p1 stride s (+ bias), then InstanceNorm3d(co, eps 1e-5, affine or not, no running stats),
                             then the activation: PReLU (one slope, init 0.25), ReLU or LeakyReLU.  Transposed: ConvTranspose3d
                             (k3, s2, p1, output_padding 1).  conv_only: the conv alone.  Keys: conv.weight, conv.bias,
                             adn.N.weight, adn.N.bias, adn.A.weight
  ResidualUnit(ci, co, s, r) conv.unit0 (stride s) .. conv.unit{r-1}, returns conv(x) + residual(x) with no activation after the
                             add; residual = Conv3d(ci, co, 3, s, p1) when s != 1, Conv3d(ci, co, 1) when only the width changes,
                             else the identity; its bias follows ``bias`` (MONAI passes bias=bias to it)
  level i, c = channels[i]   Sequential(down: inc -> c stride 2, SkipConnection(sub) -> cat([x, sub(x)], 1), up: upc -> outc);
                             sub = level i + 1 (outc = c, upc = 2c) or the bottom: a stride-1 down layer c -> channels[-1]
                             (upc = c + channels[-1]); outc of the top level = out_channels, of the others their own inc
  down layer                 ResidualUnit(subunits = num_res_units) if num_res_units > 0, else Convolution
  up layer                   Convolution(transposed, conv_only = top and num_res_units == 0), then with residual units
                             ResidualUnit(outc, outc, 1, subunits=1, last_conv_only = top)
  state dict                 depth-first registration order: model.0.*, model.1.submodule.* (recursively), model.2.*
  init                       PyTorch's defaults: conv weights and biases U(+-1/sqrt(fan_in)), PReLU 0.25
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

import torch
import torch.nn.functional as F


@dataclass
class MonaiUNetConfig:
    in_channels: int = 1
    out_channels: int = 2
    channels: Sequence[int] = (16, 32, 64, 128, 256)
    num_res_units: int = 0
    act: str = "prelu"          # "prelu", "relu" or "leakyrelu"
    act_slope: float = 0.01     # LeakyReLU's negative slope
    prelu_init: float = 0.25
    norm_affine: bool = False
    bias: bool = True


def _conv_spec(spec, cfg, pre, ci, co, transposed=False, conv_only=False):
    spec.append((pre + ".conv.weight", (ci, co, 3, 3, 3) if transposed else (co, ci, 3, 3, 3)))
    if cfg.bias:
        spec.append((pre + ".conv.bias", (co,)))
    if conv_only:
        return
    if cfg.norm_affine:
        spec += [(pre + ".adn.N.weight", (co,)), (pre + ".adn.N.bias", (co,))]
    if cfg.act == "prelu":
        spec.append((pre + ".adn.A.weight", (1,)))


def _down_spec(spec, cfg, pre, ci, co, stride):
    if cfg.num_res_units == 0:
        _conv_spec(spec, cfg, pre, ci, co)
        return
    for u in range(cfg.num_res_units):
        _conv_spec(spec, cfg, "%s.conv.unit%d" % (pre, u), ci if u == 0 else co, co)
    if stride != 1 or ci != co:
        k = 3 if stride != 1 else 1
        spec.append((pre + ".residual.weight", (co, ci, k, k, k)))
        if cfg.bias:
            spec.append((pre + ".residual.bias", (co,)))


def _up_spec(spec, cfg, pre, upc, outc, top):
    if cfg.num_res_units == 0:
        _conv_spec(spec, cfg, pre, upc, outc, transposed=True, conv_only=top)
        return
    _conv_spec(spec, cfg, pre + ".0", upc, outc, transposed=True)
    _conv_spec(spec, cfg, pre + ".1.conv.unit0", outc, outc, conv_only=top)


def _prefix(level: int) -> str:
    return "model." + "1.submodule." * level


def unet_state_dict_spec(cfg: MonaiUNetConfig) -> List[Tuple[str, Tuple[int, ...]]]:
    """Ordered (key, shape) list in MONAI's module registration order."""
    ch, L = list(cfg.channels), len(cfg.channels)
    spec: List[Tuple[str, Tuple[int, ...]]] = []

    def level(i):
        pre = _prefix(i)
        inc = cfg.in_channels if i == 0 else ch[i - 1]
        outc = cfg.out_channels if i == 0 else ch[i - 1]
        _down_spec(spec, cfg, pre + "0", inc, ch[i], 2)
        if i + 2 < L:
            level(i + 1)
            upc = 2 * ch[i]
        else:
            _down_spec(spec, cfg, pre + "1.submodule", ch[i], ch[L - 1], 1)
            upc = ch[i] + ch[L - 1]
        _up_spec(spec, cfg, pre + "2", upc, outc, i == 0)
    level(0)
    return spec


def make_unet_state_dict(cfg: MonaiUNetConfig, seed: int = 0, dtype=torch.float64) -> Dict[str, torch.Tensor]:
    """torch's default init (U(+-1/sqrt(fan_in)) for conv weights and biases), PReLU slopes at prelu_init; affine norms get
    a random weight around 1 and bias around 0 so that the tests see them"""
    g = torch.Generator().manual_seed(seed)
    spec = unet_state_dict_spec(cfg)
    shapes = dict(spec)
    out = {}
    for key, shape in spec:
        if key.endswith(".adn.A.weight"):
            out[key] = torch.full(shape, cfg.prelu_init, dtype=dtype)
        elif ".adn.N." in key:
            base = 1.0 if key.endswith("weight") else 0.0
            out[key] = (base + 0.2 * (torch.rand(shape, generator=g, dtype=torch.float64) - 0.5)).to(dtype)
        else:
            w = shapes[key[:-5] + ".weight"] if key.endswith(".bias") else shape
            bound = 1.0 / math.sqrt(w[1] * w[2] * w[3] * w[4])
            out[key] = ((torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) * bound).to(dtype)
    return out


def _act(cfg, x, sd, pre):
    if cfg.act == "prelu":
        return F.prelu(x, sd[pre + ".adn.A.weight"])
    if cfg.act == "leakyrelu":
        return F.leaky_relu(x, cfg.act_slope)
    return F.relu(x)


def _convolution(cfg, sd, pre, x, stride, transposed=False, conv_only=False):
    b = sd.get(pre + ".conv.bias")
    if transposed:
        y = F.conv_transpose3d(x, sd[pre + ".conv.weight"], b, stride=2, padding=1, output_padding=1)
    else:
        y = F.conv3d(x, sd[pre + ".conv.weight"], b, stride=stride, padding=1)
    if conv_only:
        return y
    y = F.instance_norm(y, weight=sd.get(pre + ".adn.N.weight"), bias=sd.get(pre + ".adn.N.bias"), eps=1e-5)
    return _act(cfg, y, sd, pre)


def _down(cfg, sd, pre, x, stride):
    if cfg.num_res_units == 0:
        return _convolution(cfg, sd, pre, x, stride)
    w = sd.get(pre + ".residual.weight")
    if w is not None:
        res = F.conv3d(x, w, sd.get(pre + ".residual.bias"), stride=stride, padding=1 if w.shape[2] == 3 else 0)
    else:
        res = x
    y = x
    for u in range(cfg.num_res_units):
        y = _convolution(cfg, sd, "%s.conv.unit%d" % (pre, u), y, stride if u == 0 else 1)
    return y + res


def _up(cfg, sd, pre, x, top):
    if cfg.num_res_units == 0:
        return _convolution(cfg, sd, pre, x, 2, transposed=True, conv_only=top)
    y = _convolution(cfg, sd, pre + ".0", x, 2, transposed=True)
    return _convolution(cfg, sd, pre + ".1.conv.unit0", y, 1, conv_only=top) + y


def unet_forward(x: torch.Tensor, sd: Dict[str, torch.Tensor], cfg: MonaiUNetConfig) -> torch.Tensor:
    """MONAI UNet forward in the dtype of x and sd (fp64 for the tests); differentiable with autograd"""
    L = len(cfg.channels)

    def level(i, h):
        pre = _prefix(i)
        d = _down(cfg, sd, pre + "0", h, 2)
        s = level(i + 1, d) if i + 2 < L else _down(cfg, sd, pre + "1.submodule", d, 1)
        return _up(cfg, sd, pre + "2", torch.cat([d, s], dim=1), i == 0)
    return level(0, x)
