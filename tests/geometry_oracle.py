"""fp64 CPU restatement of the geometry stage of ``augment.Compose`` (``CropForegroundd`` + ``Resized`` composed with the
spatial transforms), from the parameters a call drew (``Compose.last_params``), on top of tests/augment_oracle.py:
numpy's ``percentile_threshold`` and MONAI's ``generate_spatial_bounding_box`` restated, the composed source map
``b + s (A p) + (s - 1) / 2``, and ``F.grid_sample(align_corners=False)`` on each sample's own grid.  Independent of
csrc/foreground.cu and csrc/augment.cu."""
import numpy as np
import torch
import torch.nn.functional as F

import augment_oracle


def threshold(x: np.ndarray, p) -> np.ndarray:
    """utils/threshold.py:6-15 of the reference: np.percentile per channel of x [C][D][H][W] (fp32); None: 0 (x > 0)"""
    if p is None:
        return np.zeros(x.shape[0], dtype=x.dtype)
    return np.array([np.percentile(x[c].reshape(-1), p * 100) for c in range(x.shape[0])])


def foreground_box(x: np.ndarray, p, margin: int, allow_smaller: bool):
    """(box [3][2] (start, end), empty): the mask any_c(x_c > thr_c), then per axis the first and last selected index minus /
    plus margin, end exclusive, clipped when allow_smaller (MONAI generate_spatial_bounding_box).  An empty mask gives the
    whole volume and empty = True (MONAI: a zero-size box)."""
    thr = threshold(x, p)
    mask = (x > thr.reshape(-1, 1, 1, 1)).any(0)
    if not mask.any():
        return np.array([[0, s] for s in x.shape[1:]]), True
    box = []
    for ax in range(3):
        idx = np.nonzero(mask.any(axis=tuple(a for a in range(3) if a != ax)))[0]
        lo, hi = int(idx[0]) - margin, int(idx[-1]) + margin + 1
        if allow_smaller:
            lo, hi = max(lo, 0), min(hi, x.shape[1 + ax])
        box.append([lo, hi])
    return np.array(box), False


def source_coordinates(affine: torch.Tensor, box, out_size) -> torch.Tensor:
    """affine fp64 [3][4] on the out_size grid, box [3][2] -> source index of every output voxel, fp64 [D][H][W][3]"""
    box = torch.as_tensor(np.asarray(box), dtype=torch.float64)
    s = (box[:, 1] - box[:, 0]) / torch.tensor(out_size, dtype=torch.float64)
    ap = augment_oracle.source_coordinates(affine[None].to(torch.float64), out_size)[0]
    return box[:, 0] + s * ap + (s - 1.0) / 2.0


def sample(x: torch.Tensor, src: torch.Tensor, padding_mode: str, mode: str) -> torch.Tensor:
    """x [C][D][H][W] (any dtype) read at src [d][h][w][3] (index coordinates on x's grid) -> fp64 [C][d][h][w]"""
    size = torch.tensor(tuple(x.shape[1:]), dtype=torch.float64)
    grid = ((2.0 * src + 1.0) / size - 1.0).flip(-1)
    return F.grid_sample(x[None].to(torch.float64), grid[None], mode=mode, padding_mode=padding_mode, align_corners=False)[0]


def geometry(images, labels, params: dict):
    """The batch ``Compose`` produced for ``params`` (its ``last_params``, box on the host): fp64 image [N][C][O], fp64 label
    (or None)."""
    box = params["box"].cpu().numpy()
    out = params["spatial_size"]
    ys, ls = [], []
    for i, x in enumerate(images):
        src = source_coordinates(params["affine"][i], box[i], out)
        ys.append(sample(x, src, params["padding_mode"], "bilinear"))
        if labels is not None:
            ls.append(sample(labels[i], src, params["padding_mode"], "nearest"))
    y = augment_oracle.intensity(torch.stack(ys), params["normalize"], params["coef"])
    return y, (torch.stack(ls) if labels is not None else None)
