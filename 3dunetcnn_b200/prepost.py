"""The steps right before and right after the U-Net path, on the device (SURVEY.md section 8f, rank 4).

Mirrors (paths relative to /root/reference):
  * ``unet3d/utils/one_hot.py:7-37``   ``compile_one_hot_encoding``  label map -> one-hot uint8 target
  * ``unet3d/utils/one_hot.py:46-118`` ``convert_one_hot_to_label_map`` (+ hierarchy)  prediction -> label map
  * ``unet3d/datasets/segmentation.py:77-87``  ``normalization="zero_mean"`` -> ``monai.transforms.NormalizeIntensity``
  * ``examples/sppin/process.py:269-274``  SimpleITK ``ConnectedComponent`` + ``RelabelComponent`` -> ``connected_components``;
    ``monai.transforms.KeepLargestConnectedComponent`` -> ``keep_largest_connected_component``
  * ``unet3d/predict/volumetric.py:135-137,168-170``  ``monai.transforms.ResampleToMatch`` -> ``resample_to_match``

Same names, argument meaning and error behaviour; tensors live on the GPU and every voxel is touched by one
hand-written kernel of libb200unet instead of a chain of boolean-mask torch ops on the host.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np
import torch

from . import lib as _lib


def _plain(t: torch.Tensor) -> torch.Tensor:
    return t.as_subclass(torch.Tensor) if type(t) is not torch.Tensor else t


def _need_cuda(t: torch.Tensor, what: str) -> None:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError("%s runs only on CUDA tensors (no CPU fallback)" % what)


def compile_one_hot_encoding(data, n_labels, labels=None, dtype=torch.uint8, return_4d=True, round=True):
    """one_hot.py:7-37.  ``data``: label map (n_samples, 1, ...) -- lower-rank inputs gain leading axes; ``labels``:
    label values, a nested list groups several values into one channel; default ``1..n_labels``."""
    _need_cuda(data, "compile_one_hot_encoding")
    x = _plain(data)
    while x.dim() < 5:
        x = x[None]
    assert x.shape[1] == 1
    if dtype != torch.uint8:
        raise NotImplementedError("compile_one_hot_encoding: only dtype=torch.uint8 (the reference's default) is implemented")
    values, begin = [], [0]
    for i in range(n_labels):
        if labels is not None:
            group = labels[i] if type(labels[i]) == list else [labels[i]]
        else:
            group = [i + 1]
        values.extend(float(v) for v in group)
        begin.append(len(values))
    x = x.contiguous().float()
    n = x.shape[0]
    spatial = x[0, 0].numel()
    y = torch.empty((n, n_labels) + tuple(x.shape[2:]), dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load_library().b200unet_one_hot(x.data_ptr(), n, spatial, (C.c_float * len(values))(*values),
                                                        (C.c_int32 * len(begin))(*begin), n_labels, int(bool(round)),
                                                        y.data_ptr(), _lib.stream_ptr()), "one_hot")
    if return_4d:
        assert y.shape[0] == 1
        y = y[0]
    return y


def normalize_intensity(img: torch.Tensor, nonzero: bool = False, channel_wise: bool = False,
                        subtrahend=None, divisor=None) -> torch.Tensor:
    """``monai.transforms.NormalizeIntensity`` on one channel-first image (C, ...): ``(img - mean) / std`` (population
    std; ``std == 0`` -> 1), per channel when ``channel_wise``; ``nonzero``: statistics over, and changes to, the
    non-zero voxels only.  Parity unpinned (MONAI absent): restated from its documented behaviour."""
    _need_cuda(img, "normalize_intensity")
    if subtrahend is not None or divisor is not None:
        raise NotImplementedError("normalize_intensity: explicit subtrahend/divisor are not implemented")
    x = _plain(img).contiguous().float()
    groups = x.shape[0] if channel_wise else 1
    spatial = x.numel() // groups
    y = torch.empty_like(x)
    stats = torch.empty((groups, 3), dtype=torch.float64, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load_library().b200unet_zscore(x.data_ptr(), groups, spatial, int(bool(nonzero)), stats.data_ptr(),
                                                       y.data_ptr(), _lib.stream_ptr()), "zscore")
    return y


def _label_map(p: torch.Tensor, labels: Sequence[int], act: int, threshold: float, hierarchy: bool, sum_then_threshold: bool):
    x = p.contiguous().float()
    L = len(labels)
    if x.shape[0] < L:
        raise ValueError("one-hot encoding has %d channels but %d labels were given" % (x.shape[0], L))
    spatial = x[0].numel()
    out = torch.empty(tuple(x.shape[1:]), dtype=torch.int16, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load_library().b200unet_label_map(x.data_ptr(), L, spatial, (C.c_int32 * L)(*[int(v) for v in labels]), act,
                                                          float(threshold), int(bool(hierarchy)), int(bool(sum_then_threshold)),
                                                          out.data_ptr(), _lib.stream_ptr()), "label_map")
    return out


_ACT = {None: 0, "sigmoid": 1, "softmax": 2}


def convert_one_hot_to_label_map(one_hot_encoding, labels, axis=0, threshold=0.5, sum_then_threshold=False,
                                 dtype=torch.int16, label_hierarchy=False, activation: Optional[str] = None):
    """one_hot.py:46-67 on a channel-first prediction (L, ...).  ``activation`` (extension): apply sigmoid / softmax
    to logits inside the same kernel (volumetric.py:151-156 runs it as a separate pass)."""
    _need_cuda(one_hot_encoding, "convert_one_hot_to_label_map")
    if axis != 0:
        raise NotImplementedError("convert_one_hot_to_label_map: only axis=0 (channel first) is implemented")
    if dtype != torch.int16:
        raise NotImplementedError("convert_one_hot_to_label_map: only dtype=torch.int16 (the reference's default)")
    if activation not in _ACT:
        raise ValueError("activation must be None, 'sigmoid' or 'softmax'")
    x = _plain(one_hot_encoding)
    if label_hierarchy:
        return _label_map(x, labels, _ACT[activation], threshold, True, False)
    if all(type(_labels) == list for _labels in labels):
        # several label-map volumes, one per group of channels (one_hot.py:53-62); the activation spans all channels, so
        # it is applied per group only when it is channel-independent
        if activation == "softmax":
            raise NotImplementedError("softmax across grouped label maps: apply it before the call")
        maps, i = [], 0
        for _labels in labels:
            maps.append(_label_map(x[i:i + len(_labels)], _labels, _ACT[activation], threshold, False, sum_then_threshold))
            i += len(_labels)
        return torch.stack(maps, dim=axis)
    return _label_map(x, labels, _ACT[activation], threshold, False, sum_then_threshold)


def convert_one_hot_to_label_map_using_hierarchy(one_hot_encoding, labels, threshold=0.5, axis=0, dtype=torch.int16):
    """one_hot.py:92-110."""
    return convert_one_hot_to_label_map(one_hot_encoding, labels, axis=axis, threshold=threshold, dtype=dtype,
                                        label_hierarchy=True)


def _check_connectivity(connectivity) -> int:
    if isinstance(connectivity, bool) or connectivity not in (1, 2, 3):
        raise ValueError("connectivity must be 1 (6 face neighbours), 2 (18) or 3 (26), got %r" % (connectivity,))
    return int(connectivity)


def _size_ordered_labels(m8: torch.Tensor, connectivity: int):
    """m8 uint8 [nvol, d, h, w] -> (int32 labels numbered by decreasing size, CPU int32 counts [nvol]).  The counts are the one
    device-to-host read: their maximum sizes the sort."""
    m8 = m8.contiguous()                         # the kernels read a C-order [nvol, d, h, w] array
    nvol, d, h, w = m8.shape
    labels = torch.empty(m8.shape, dtype=torch.int32, device=m8.device)
    counts = torch.empty(nvol, dtype=torch.int32, device=m8.device)
    with torch.cuda.device(m8.device):
        scratch = torch.empty(_lib.cc_scratch_bytes(nvol, d, h, w), dtype=torch.uint8, device=m8.device)
        _lib.cc_label(m8, connectivity, labels, counts, scratch)
        counts = counts.cpu()
        _lib.cc_sort_by_size(labels, int(counts.max()), scratch)
    return labels, counts


def connected_components(mask: torch.Tensor, connectivity: int = 1):
    """Label the connected components of a mask (..., D, H, W) on the device: nonzero is foreground, every leading index is an
    independent volume, ``connectivity`` counts orthogonal hops (1 = 6 face neighbours, 2 = 18, 3 = 26) as in scipy and MONAI.

    Returns ``(labels, counts)``: int32 labels of the mask's shape, 0 for background and 1..K numbered by decreasing component
    size, equal sizes in raster order of their first voxel (SimpleITK ``ConnectedComponent`` followed by
    ``RelabelComponent(sortByObjectSize=True)``), and K per volume as a CPU int64 tensor over the leading dimensions.  So the
    largest component of a prediction is ``connected_components(pred > 0.5)[0] == 1``.  Exact: no tolerance, the same result
    every run.  One device-to-host read (the counts)."""
    connectivity = _check_connectivity(connectivity)
    _need_cuda(mask, "connected_components")
    m = _plain(mask)
    if m.dim() < 3:
        raise ValueError("connected_components: expected a mask (..., D, H, W), got shape %s" % (tuple(m.shape),))
    lead, (d, h, w) = tuple(m.shape[:-3]), tuple(m.shape[-3:])
    if m.numel() == 0:
        return torch.zeros(m.shape, dtype=torch.int32, device=m.device), torch.zeros(lead, dtype=torch.int64)
    if m.dtype == torch.uint8:
        m8 = m
    elif m.dtype == torch.bool:
        m8 = m.view(torch.uint8)
    else:
        m8 = (m != 0).view(torch.uint8)
    labels, counts = _size_ordered_labels(m8.reshape(-1, d, h, w), connectivity)
    return labels.reshape(m.shape), counts.to(torch.int64).reshape(lead)


def keep_largest_connected_component(img: torch.Tensor, applied_labels=None, is_onehot: Optional[bool] = None,
                                     independent: bool = True, connectivity: Optional[int] = None, num_components: int = 1):
    """``monai.transforms.KeepLargestConnectedComponent`` on a channel-first 3D image (C, D, H, W) on the device.

    ``img`` is a label map (one channel) or a one-hot image; ``is_onehot`` None means C > 1.  ``applied_labels``: the label
    values (label map) or channels (one-hot) to clean; None means every label value but 0, or every channel but 0.
    ``independent``: clean each applied label on its own; otherwise their union is one foreground.  ``connectivity`` in orthogonal
    hops (None = 3, the 26-neighbourhood); ``num_components`` components are kept.  Foreground voxels of the other components
    are set to 0 in a new tensor of the input's dtype; the input is not modified.

    Components are ranked by size, equal sizes in raster order of their first voxel (SimpleITK's ``RelabelComponent`` order).
    MONAI ranks equal sizes with an unstable ``argsort``, so where components of equal size straddle the ``num_components``
    cut the kept one may differ from MONAI's; everywhere else the result is MONAI's.  At most two device-to-host reads: the
    component counts, and the label values when ``applied_labels`` is None on a label map."""
    connectivity = _check_connectivity(3 if connectivity is None else connectivity)
    _need_cuda(img, "keep_largest_connected_component")
    x = _plain(img)
    if x.dim() != 4:
        raise ValueError("keep_largest_connected_component: expected a channel-first 3D image (C, D, H, W), got shape %s"
                         % (tuple(x.shape),))
    if x.numel() == 0:
        return x.clone()
    onehot = x.shape[0] > 1 if is_onehot is None else bool(is_onehot)
    if applied_labels is not None:
        applied = list(applied_labels) if isinstance(applied_labels, (list, tuple)) else [applied_labels]
    elif onehot:
        # MONAI takes the channels holding any foreground, minus 0; a channel without foreground changes nothing
        applied = list(range(1, x.shape[0]))
    else:
        if x.shape[0] != 1:
            raise ValueError("If input not one-hotted, should only be 1 channel, got %d." % x.shape[0])
        applied = [v for v in torch.unique(x).tolist() if v != 0]
    out = x.clone()
    if not applied:
        return out
    if onehot:
        idx = [int(i) for i in applied]
        fg = x[idx] > 0 if independent else (x[idx] == 1).any(0, keepdim=True)
    else:
        fg = torch.stack([x[0] == v for v in applied])
        if not independent:
            fg = fg.any(0, keepdim=True)
    labels, _ = _size_ordered_labels(fg.view(torch.uint8), connectivity)
    drop = fg & (labels > num_components)
    if onehot:
        out[idx] = out[idx].masked_fill(drop, 0)
    else:
        out[0].masked_fill_(drop.any(0), 0)      # the label masks are disjoint
    return out


# MONAI's resolves_modes maps every *linear mode to grid_sample's bilinear, which is trilinear on a volume
_RESAMPLE_MODES = {"trilinear": 0, "bilinear": 0, "linear": 0, "nearest": 1}
# An index-map entry within this distance of an integer is taken as that integer.  A crop, flip or axis permutation composed
# from inexact voxel spacings (or from affines stored in fp32) then copies voxels exactly instead of blending in a 1e-12 share
# of a neighbour, and two grids whose index map is the identity to this tolerance count as equal (the resample is skipped).
INDEX_MAP_TOL = 1e-6


def resample_mode(mode) -> int:
    """the kernel's mode for an ``interpolation`` / ``mode`` argument: 0 trilinear, 1 nearest"""
    if isinstance(mode, str) and mode in _RESAMPLE_MODES:
        return _RESAMPLE_MODES[mode]
    raise NotImplementedError("resample_to_match: mode %r is not implemented; use 'trilinear' (or 'bilinear' / 'linear', the same "
                              "on a volume) or 'nearest'" % (mode,))


def _affines(a, n: int, what: str):
    """a [4, 4] affine shared by all n items, or one per item [n, 4, 4] -> list of n fp64 arrays"""
    if isinstance(a, torch.Tensor):
        a = _plain(a).detach().cpu().double().numpy()
    a = np.asarray(a, dtype=np.float64)
    if a.shape == (4, 4):
        return [a] * n
    if a.shape == (n, 4, 4):
        return list(a)
    raise ValueError("resample_to_match: %s must be a 4x4 affine or one per item [%d, 4, 4], got shape %s" % (what, n, a.shape))


def index_map(src_affine, dst_affine) -> np.ndarray:
    """fp64 3x4 map of a target voxel index (d, h, w, 1) to the source index: inv(src_affine) @ dst_affine, voxel centres on
    integers (MONAI's spatial_resample with normalized=False).  Entries within INDEX_MAP_TOL of an integer are snapped to it."""
    m = np.linalg.solve(np.asarray(src_affine, dtype=np.float64), np.asarray(dst_affine, dtype=np.float64))[:3]
    r = np.rint(m)
    return np.where(np.abs(m - r) <= INDEX_MAP_TOL, r, m)


def resample_to_match(img: torch.Tensor, src_affine, dst_affine, dst_shape, mode: str = "trilinear") -> torch.Tensor:
    """``monai.transforms.ResampleToMatch(mode)`` as volumetric.py:135-137,168-170 calls it, on the device: resample a channel-first
    image ``[C, D, H, W]`` (or a batch ``[N, C, D, H, W]``) whose grid has the affine ``src_affine`` onto the grid of shape
    ``dst_shape`` with the affine ``dst_affine`` (4x4 voxel-to-world; either may be one per item ``[N, 4, 4]``).  Returns fp32
    ``[C, *dst_shape]`` (``[N, C, *dst_shape]``).  Parity unpinned: MONAI is absent from this image.

    ``mode``: 'trilinear', 'bilinear' or 'linear' (all trilinear on a volume), or 'nearest' (round half to even, as
    grid_sample); anything else raises ``NotImplementedError``.  Padding is MONAI's default, border: target voxels that map
    outside the source take the nearest edge value (so outside a foreground crop the prediction's edge extends to the volume
    boundary, as the reference writes it).  When the shapes are equal and ``index_map`` is the identity (affines equal to
    INDEX_MAP_TOL) the image is copied unchanged.  One kernel per item, no CPU fallback."""
    m = resample_mode(mode)
    _need_cuda(img, "resample_to_match")
    x = _plain(img)
    if x.dim() not in (4, 5):
        raise ValueError("resample_to_match: expected [C, D, H, W] or [N, C, D, H, W], got shape %s" % (tuple(x.shape),))
    xs = (x if x.dim() == 5 else x[None]).contiguous().float()
    n, c = xs.shape[:2]
    src, dst = _affines(src_affine, n, "src_affine"), _affines(dst_affine, n, "dst_affine")
    shape = tuple(int(s) for s in (dst_shape.tolist() if hasattr(dst_shape, "tolist") else dst_shape))
    if len(shape) != 3 or min(shape) < 1:
        raise ValueError("resample_to_match: dst_shape must be three positive extents, got %r" % (dst_shape,))
    out = torch.empty((n, c) + shape, dtype=torch.float32, device=xs.device)
    identity = np.eye(4)[:3]
    lib = _lib.load_library()
    with torch.cuda.device(xs.device):
        for i in range(n):
            a = index_map(src[i], dst[i])
            if shape == tuple(xs.shape[2:]) and np.array_equal(a, identity):
                out[i].copy_(xs[i])
                continue
            _lib.check(lib.b200unet_resample_to_grid(xs[i].data_ptr(), c, *xs.shape[2:], (C.c_double * 12)(*a.ravel().tolist()), m,
                                                     out[i].data_ptr(), *shape, _lib.stream_ptr()), "resample_to_grid")
    return out if x.dim() == 5 else out[0]
