"""CPU restatement of the reference ``UNet3D`` forward, the MONAI Dice criterion
and the MONAI sliding-window inferer.  TEST INFRASTRUCTURE ONLY (see
``oracle/__init__.py``).

Every function cites the reference file:line (relative to /root/reference) it
restates.  The arithmetic library is torch's CPU ``torch.nn.functional`` --
the same third-party library the reference dispatches to (SURVEY.md 8c) --
plus plain-numpy restatements of the three stencil ops used to cross-check it.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------
# configuration  (unet3d/models/pytorch/autoencoder/variational.py:38-41, segmentation/unet.py:48)
# --------------------------------------------------------------------------------------
@dataclass
class UNetConfig:
    n_features: int = 1
    n_outputs: int = 1
    base_width: int = 32
    encoder_blocks: Sequence[int] = (1, 2, 2, 4)
    decoder_blocks: Optional[Sequence[int]] = None  # None -> [1]*len(encoder_blocks) (variational.py:75-76)
    feature_dilation: int = 2
    downsampling_stride: int = 2
    use_transposed_convolutions: bool = False
    kernel_size: int = 3
    layer_widths: Optional[Sequence[int]] = None
    norm_groups: int = 8            # myronenko.py:6
    dropout: float = 0.2            # myronenko.py:85 (hard-wired, level 0 only)
    activation: Optional[str] = None
    interpolation_mode: str = "trilinear"

    def enc_widths(self) -> List[int]:
        # myronenko.py:94-97
        if self.layer_widths is not None:
            return list(self.layer_widths[: len(self.encoder_blocks)])
        return [self.base_width * self.feature_dilation ** i for i in range(len(self.encoder_blocks))]

    def dec_blocks(self) -> List[int]:
        return list(self.decoder_blocks) if self.decoder_blocks is not None else [1] * len(self.encoder_blocks)

    def dec_widths(self, depth: int) -> Tuple[int, int]:
        """(in_width, out_width) of decoder stage ``depth`` -- decoder.py:111-122 + unet.py:20-25."""
        n = len(self.dec_blocks())
        if self.layer_widths is not None:
            out_w = self.layer_widths[depth]
            in_w = self.layer_widths[depth + 1] if depth + 1 < len(self.layer_widths) else self.layer_widths[depth]
        elif depth > 0:
            out_w = int(self.base_width * self.feature_dilation ** (depth - 1))
            in_w = out_w * self.feature_dilation
        else:
            out_w = self.base_width
            in_w = self.base_width
        if depth != n - 1:
            in_w *= 2
        return in_w, out_w


def _groups(c: int, norm_groups: int) -> int:
    # myronenko.py:23-31
    if c < norm_groups or c % norm_groups:
        return c
    return norm_groups


def unet3d_state_dict_spec(cfg: UNetConfig) -> List[Tuple[str, Tuple[int, ...]]]:
    """Ordered (key, shape) list of the reference ``UNet3D.state_dict()`` (SURVEY.md appendix B)."""
    k = cfg.kernel_size
    spec: List[Tuple[str, Tuple[int, ...]]] = []

    def block(prefix: str, cin: int, cout: int):
        spec.append((f"{prefix}.conv1.norm1.weight", (cin,)))
        spec.append((f"{prefix}.conv1.norm1.bias", (cin,)))
        spec.append((f"{prefix}.conv1.conv.weight", (cout, cin, k, k, k)))
        spec.append((f"{prefix}.conv2.norm1.weight", (cout,)))
        spec.append((f"{prefix}.conv2.norm1.bias", (cout,)))
        spec.append((f"{prefix}.conv2.conv.weight", (cout, cout, k, k, k)))
        if cin != cout:
            spec.append((f"{prefix}.sample.weight", (cout, cin, 1, 1, 1)))

    widths = cfg.enc_widths()
    cin = cfg.n_features
    for li, nb in enumerate(cfg.encoder_blocks):
        c = widths[li]
        for b in range(nb):
            block(f"encoder.layers.{li}.blocks.{b}", cin if b == 0 else c, c)
        cin = c
    for li in range(len(cfg.encoder_blocks) - 1):
        c = widths[li]
        spec.append((f"encoder.downsampling_convolutions.{li}.weight", (c, c, k, k, k)))

    dblocks = cfg.dec_blocks()
    n = len(dblocks)
    ups = []
    for i, nb in enumerate(dblocks):
        depth = n - (i + 1)
        in_w, out_w = cfg.dec_widths(depth)
        planes = in_w if depth != 0 else out_w
        for b in range(nb):
            block(f"decoder.layers.{i}.blocks.{b}", in_w if b == 0 else planes, planes)
        if depth != 0:
            ups.append((i, in_w, out_w))
    if cfg.use_transposed_convolutions:
        for i, in_w, out_w in ups:
            spec.append((f"decoder.upsampling_blocks.{i}.weight", (in_w, out_w, k, k, k)))
            spec.append((f"decoder.upsampling_blocks.{i}.bias", (out_w,)))
    else:
        for i, in_w, out_w in ups:
            spec.append((f"decoder.pre_upsampling_blocks.{i}.weight", (out_w, in_w, 1, 1, 1)))
    spec.append(("final_convolution.weight", (cfg.n_outputs, cfg.base_width, 1, 1, 1)))
    return spec


def make_state_dict(cfg: UNetConfig, seed: int = 0, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """Deterministic weights independent of module construction order.

    conv weights ~ U(+-1/sqrt(fan_in)) like torch's default Conv3d init (SURVEY appendix B);
    norm gamma ~ 1 + 0.2*N(0,1), beta ~ 0.1*N(0,1) so the affine path is exercised.
    Each tensor draws from its own generator seeded by (seed, index) -> stable under reordering.
    """
    out: Dict[str, torch.Tensor] = {}
    for idx, (key, shape) in enumerate(unet3d_state_dict_spec(cfg)):
        g = torch.Generator().manual_seed(1000003 * (seed + 1) + idx)
        if key.endswith("norm1.weight"):
            t = 1.0 + 0.2 * torch.randn(shape, generator=g, dtype=torch.float64)
        elif key.endswith("norm1.bias"):
            t = 0.1 * torch.randn(shape, generator=g, dtype=torch.float64)
        elif key.endswith(".bias"):
            t = 0.1 * (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1)
        else:
            if "upsampling_blocks" in key and not key.startswith("decoder.pre"):
                fan_in = shape[1] * int(np.prod(shape[2:]))  # ConvTranspose3d: weight.size(1)*k^3
            else:
                fan_in = shape[1] * int(np.prod(shape[2:]))
            bound = 1.0 / math.sqrt(fan_in)
            t = (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) * bound
        out[key] = t.to(dtype)
    return out


# --------------------------------------------------------------------------------------
# forward restatement
# --------------------------------------------------------------------------------------
def _conv_block(sd, prefix, x, cfg: UNetConfig, stride=1, slope: float = 0.0):
    # myronenko.py:17-21  GN -> ReLU -> conv (bias-free, padding=k//2: resnet.py:12-17)
    cin = x.shape[1]
    x = F.group_norm(x, _groups(cin, cfg.norm_groups), sd[f"{prefix}.norm1.weight"], sd[f"{prefix}.norm1.bias"], eps=1e-5)
    x = F.relu(x) if slope == 0.0 else F.leaky_relu(x, slope)
    return F.conv3d(x, sd[f"{prefix}.conv.weight"], None, stride=stride, padding=cfg.kernel_size // 2)


def _res_block(sd, prefix, x, cfg: UNetConfig, slope: float = 0.0):
    # myronenko.py:47-58
    identity = x
    y = _conv_block(sd, f"{prefix}.conv1", x, cfg, slope=slope)
    y = _conv_block(sd, f"{prefix}.conv2", y, cfg, slope=slope)
    if f"{prefix}.sample.weight" in sd:
        identity = F.conv3d(identity, sd[f"{prefix}.sample.weight"])
    return y + identity


def _layer(sd, prefix, x, n_blocks, cfg, dropout_mask=None, slope: float = 0.0):
    # myronenko.py:75-80 ; Dropout3d after block 0 (level 0 of the encoder only, myronenko.py:97-100)
    for b in range(n_blocks):
        x = _res_block(sd, f"{prefix}.blocks.{b}", x, cfg, slope)
        if b == 0 and dropout_mask is not None:
            x = x * dropout_mask.to(x.dtype).view(x.shape[0], x.shape[1], 1, 1, 1)
    return x


def unet3d_forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, cfg: UNetConfig,
                   dropout_mask: Optional[torch.Tensor] = None, return_intermediates: bool = False,
                   slope: float = 0.0):
    """Reference ``UNet3D.forward`` (variational.py:81-87 -> unet.py:8-16 -> unet.py:27-44).

    ``dropout_mask``: optional (N, C0) tensor of per-channel scales (0 or 1/(1-p)) applied after
    block 0 of encoder level 0 -- Dropout3d semantics (SURVEY appendix C).  None == eval mode.
    ``slope``: negative slope of the activation after each GroupNorm; 0 is the reference's ReLU.  Slope 1 makes
    the network smooth, so its gradients can be compared at tight bounds (tests/plan_smooth_cases.py).
    """
    nlev = len(cfg.encoder_blocks)
    skips = []
    inter = {}
    for li, nb in enumerate(cfg.encoder_blocks):
        x = _layer(sd, f"encoder.layers.{li}", x, nb, cfg, dropout_mask if li == 0 else None, slope)
        skips.insert(0, x)  # unet.py:12
        if li != nlev - 1:
            x = F.conv3d(x, sd[f"encoder.downsampling_convolutions.{li}.weight"], None,
                         stride=cfg.downsampling_stride, padding=cfg.kernel_size // 2)  # unet.py:13
    inter["bottleneck"] = skips[0]
    dblocks = cfg.dec_blocks()
    x = skips[0]
    for i in range(len(dblocks) - 1):
        x = _layer(sd, f"decoder.layers.{i}", x, dblocks[i], cfg, slope=slope)  # unet.py:30
        if cfg.use_transposed_convolutions:
            x = F.conv_transpose3d(x, sd[f"decoder.upsampling_blocks.{i}.weight"],
                                   sd[f"decoder.upsampling_blocks.{i}.bias"],
                                   stride=cfg.downsampling_stride, padding=1)  # decoder.py:101-102
        else:
            x = F.conv3d(x, sd[f"decoder.pre_upsampling_blocks.{i}.weight"])  # decoder.py:104
            x = F.interpolate(x, scale_factor=cfg.downsampling_stride, mode=cfg.interpolation_mode,
                              align_corners=False)                              # decoder.py:105-106
        skip = skips[i + 1]
        dz = skip.shape[2] - x.shape[2]
        dy = skip.shape[3] - x.shape[3]
        dx = skip.shape[4] - x.shape[4]
        x = F.pad(x, [dx // 2, dx - dx // 2, dy // 2, dy - dy // 2, dz // 2, dz - dz // 2])  # unet.py:34-40
        x = torch.cat((x, skip), 1)                                                       # unet.py:42
    x = _layer(sd, f"decoder.layers.{len(dblocks) - 1}", x, dblocks[-1], cfg, slope=slope)  # unet.py:43
    inter["decoder_out"] = x
    x = F.conv3d(x, sd["final_convolution.weight"])                                       # variational.py:84
    if cfg.activation == "sigmoid":
        x = torch.sigmoid(x)
    elif cfg.activation == "softmax":
        x = torch.softmax(x, dim=1)
    if return_intermediates:
        return x, inter
    return x


# --------------------------------------------------------------------------------------
# Dice criterion  (monai.losses.DiceLoss restated from its public definition; call site
# unet3d/scripts/script_utils.py:61-77, config examples/brats2020/brats2020_config.json:112-116)
# --------------------------------------------------------------------------------------
def dice_loss(logits: torch.Tensor, target: torch.Tensor, *, sigmoid: bool = True, softmax: bool = False,
              include_background: bool = True, squared_pred: bool = False, jaccard: bool = False,
              batch: bool = False, reduction: str = "mean", smooth_nr: float = 1e-5,
              smooth_dr: float = 1e-5) -> torch.Tensor:
    p = logits
    if sigmoid:
        p = torch.sigmoid(p)
    if softmax:
        p = torch.softmax(p, dim=1)
    t = target.to(p.dtype)
    if not include_background and p.shape[1] > 1:
        p = p[:, 1:]
        t = t[:, 1:]
    axes = list(range(2, p.dim()))
    if batch:
        axes = [0] + axes
    inter = (p * t).sum(dim=axes)
    if squared_pred:
        ground = (t * t).sum(dim=axes)
        pred = (p * p).sum(dim=axes)
    else:
        ground = t.sum(dim=axes)
        pred = p.sum(dim=axes)
    denom = ground + pred
    if jaccard:
        denom = 2.0 * (denom - inter)
    f = 1.0 - (2.0 * inter + smooth_nr) / (denom + smooth_dr)
    if reduction == "mean":
        return f.mean()
    if reduction == "sum":
        return f.sum()
    return f


def dice_loss_grad(logits: torch.Tensor, target: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """Closed-form d(mean Dice)/d(logits) for sigmoid=True, include_background=True (SURVEY appendix C)."""
    p = torch.sigmoid(logits)
    t = target.to(p.dtype)
    axes = list(range(2, p.dim()))
    I = (p * t).sum(dim=axes, keepdim=True)
    P = p.sum(dim=axes, keepdim=True)
    T = t.sum(dim=axes, keepdim=True)
    D = P + T + eps
    nc = logits.shape[0] * logits.shape[1]
    return -(2.0 * t * D - (2.0 * I + eps)) / (D * D) * p * (1.0 - p) / nc


# --------------------------------------------------------------------------------------
# sliding window inferer (monai.inferers.SlidingWindowInferer restated; call sites
# unet3d/scripts/script_utils.py:290-293, unet3d/predict/volumetric.py:147-148)   -- parity unpinned
# --------------------------------------------------------------------------------------
def _scan_starts(size: int, roi: int, overlap: float) -> List[int]:
    interval = max(int(roi * (1 - overlap)), 1)
    if size <= roi:
        return [0]
    n = int(math.ceil(float(size - roi) / interval)) + 1
    return [min(i * interval, size - roi) for i in range(n)]


def gaussian_importance(roi: Sequence[int], sigma_scale: float = 0.125) -> torch.Tensor:
    w = None
    for r in roi:
        c = (r - 1) / 2.0
        s = sigma_scale * r
        g = torch.exp(-0.5 * ((torch.arange(r, dtype=torch.float32) - c) / s) ** 2)
        w = g if w is None else w[..., None] * g
    w = w / w.max()
    mn = w[w > 0].min()
    return torch.clamp(w, min=float(mn))


def sliding_window_inference(x: torch.Tensor, roi: Sequence[int], predictor, overlap: float = 0.25,
                             mode: str = "constant", sw_batch_size: int = 1) -> torch.Tensor:
    n, _, D, H, W = x.shape
    roi = [min(r, s) for r, s in zip(roi, (D, H, W))]
    w = torch.ones(roi) if mode == "constant" else gaussian_importance(roi)
    out = None
    cnt = torch.zeros((1, 1, D, H, W), dtype=torch.float32)
    windows = [(d, h, ww) for d in _scan_starts(D, roi[0], overlap) for h in _scan_starts(H, roi[1], overlap)
               for ww in _scan_starts(W, roi[2], overlap)]
    for (d, h, ww) in windows:
        patch = x[:, :, d:d + roi[0], h:h + roi[1], ww:ww + roi[2]]
        pred = predictor(patch)
        if out is None:
            out = torch.zeros((n, pred.shape[1], D, H, W), dtype=torch.float32)
        out[:, :, d:d + roi[0], h:h + roi[1], ww:ww + roi[2]] += pred.float() * w
        cnt[:, :, d:d + roi[0], h:h + roi[1], ww:ww + roi[2]] += w
    return out / cnt


# --------------------------------------------------------------------------------------
# plain-numpy restatements of the stencil ops (used to cross-check torch's CPU kernels)
# --------------------------------------------------------------------------------------
def conv3d_direct(x: np.ndarray, w: np.ndarray, stride: int = 1, padding: int = 1) -> np.ndarray:
    """Cross-correlation, zero padding, no bias (SURVEY appendix C). x:[N,C,D,H,W] w:[O,C,k,k,k]."""
    n, c, D, H, W = x.shape
    o, _, k, _, _ = w.shape
    xp = np.pad(x.astype(np.float64), ((0, 0), (0, 0)) + ((padding, padding),) * 3)
    Do = (D + 2 * padding - k) // stride + 1
    Ho = (H + 2 * padding - k) // stride + 1
    Wo = (W + 2 * padding - k) // stride + 1
    y = np.zeros((n, o, Do, Ho, Wo), dtype=np.float64)
    for kd in range(k):
        for kh in range(k):
            for kw in range(k):
                patch = xp[:, :, kd:kd + stride * Do:stride, kh:kh + stride * Ho:stride, kw:kw + stride * Wo:stride]
                y += np.einsum("ncdhw,oc->nodhw", patch, w[:, :, kd, kh, kw].astype(np.float64))
    return y


def group_norm(x: np.ndarray, groups: int, gamma: np.ndarray, beta: np.ndarray, eps: float = 1e-5) -> np.ndarray:
    n, c = x.shape[:2]
    xr = x.astype(np.float64).reshape(n, groups, -1)
    mu = xr.mean(axis=2, keepdims=True)
    var = xr.var(axis=2, keepdims=True)  # biased
    y = ((xr - mu) / np.sqrt(var + eps)).reshape(x.shape)
    shp = (1, c) + (1,) * (x.ndim - 2)
    return y * gamma.reshape(shp) + beta.reshape(shp)


def _up1d(x: np.ndarray, axis: int) -> np.ndarray:
    n = x.shape[axis]
    idx = np.arange(2 * n)
    src = (idx + 0.5) / 2.0 - 0.5
    src = np.clip(src, 0, None)
    i0 = np.floor(src).astype(int)
    i1 = np.minimum(i0 + 1, n - 1)
    lam = src - i0
    a = np.take(x, i0, axis=axis)
    b = np.take(x, i1, axis=axis)
    shp = [1] * x.ndim
    shp[axis] = 2 * n
    lam = lam.reshape(shp)
    return a * (1 - lam) + b * lam


def trilinear_upsample2x(x: np.ndarray) -> np.ndarray:
    """F.interpolate(scale_factor=2, mode='trilinear', align_corners=False) restated (SURVEY appendix C)."""
    y = x.astype(np.float64)
    for ax in (2, 3, 4):
        y = _up1d(y, ax)
    return y
