"""CPU restatement of MONAI's boundary-distance metrics (monai/metrics/utils.py get_mask_edges / get_surface_distance,
hausdorff_distance.py, surface_distance.py, surface_dice.py of MONAI 1.3+), in numpy with scipy.ndimage.binary_erosion /
distance_transform_edt and torch.quantile in fp32, as MONAI calls them.  MONAI crops both masks to their union box (plus a
background margin) before the erosion; that changes no edge and no distance, so the oracle works on the whole volume.

Empty masks follow MONAI's arrays: both empty -> no distances (nan); exactly one empty -> arrays of inf (HD and ASD inf, NSD 0).
torch.quantile of an all-inf array is nan (its lerp computes inf - inf); the oracle returns the inf that array stands for.
ASD is returned as the fp64 mean of the concatenated fp32 distances (MONAI's fp32 torch.mean rounds it once more).
"""
import numpy as np
import torch
from scipy import ndimage


def edges(mask: np.ndarray) -> np.ndarray:
    """fg & ~erode(fg): 6-neighbour cross, outside = background (scipy's defaults)"""
    mask = np.asarray(mask, dtype=bool)
    if not mask.any():
        return np.zeros_like(mask)
    return mask & ~ndimage.binary_erosion(mask)


def surface_distance(e_pred: np.ndarray, e_gt: np.ndarray, spacing) -> np.ndarray:
    """MONAI get_surface_distance on edge masks: fp32 distances from each e_pred voxel to the nearest e_gt voxel"""
    if not e_gt.any():
        return np.full(int(e_pred.sum()), np.inf, dtype=np.float32)
    if not e_pred.any():
        return np.full(int(e_gt.sum()), np.inf, dtype=np.float32)
    dis = ndimage.distance_transform_edt(~e_gt, sampling=spacing)
    return dis.astype(np.float32)[e_pred]


def foreground(x) -> np.ndarray:
    """MONAI's label_idx = 1 after the cast to float"""
    return np.asarray(torch.as_tensor(x).detach().cpu().float().numpy() == 1.0)


def pair_distances(pred, gt, spacing=None, symmetric=True):
    ep, eg = edges(foreground(pred)), edges(foreground(gt))
    d = [surface_distance(ep, eg, spacing)]
    if symmetric:
        d.append(surface_distance(eg, ep, spacing))
    return d


def _percentile(d: np.ndarray, percentile):
    if d.size == 0:
        return np.float32(np.nan)
    if np.isinf(d).all():
        return np.float32(np.inf)
    t = torch.from_numpy(d)
    if not percentile:
        return np.float32(t.max().item())
    return np.float32(torch.quantile(t, percentile / 100).item())


def _spacing_list(spacing, b):
    if spacing is None or isinstance(spacing, (int, float)):
        return [spacing] * b
    if isinstance(spacing[0], (int, float)):
        return [spacing] * b
    return list(spacing)


def _drop_bg(x, include_background):
    x = torch.as_tensor(x)
    return x if include_background or x.shape[1] == 1 else x[:, 1:]


def hausdorff(y_pred, y, include_background=False, percentile=None, directed=False, spacing=None) -> np.ndarray:
    y_pred, y = _drop_bg(y_pred, include_background), _drop_bg(y, include_background)
    b, c = y_pred.shape[:2]
    sp = _spacing_list(spacing, b)
    out = np.empty((b, c), np.float32)
    for i in range(b):
        for j in range(c):
            ds = pair_distances(y_pred[i, j], y[i, j], sp[i], symmetric=not directed)
            out[i, j] = np.float32(torch.max(torch.tensor([_percentile(d, percentile) for d in ds])).item())
    return out


def average_surface(y_pred, y, include_background=False, symmetric=False, spacing=None) -> np.ndarray:
    """fp64 [B, C'] means"""
    y_pred, y = _drop_bg(y_pred, include_background), _drop_bg(y, include_background)
    b, c = y_pred.shape[:2]
    sp = _spacing_list(spacing, b)
    out = np.empty((b, c), np.float64)
    for i in range(b):
        for j in range(c):
            d = np.concatenate(pair_distances(y_pred[i, j], y[i, j], sp[i], symmetric=symmetric))
            out[i, j] = np.nan if d.size == 0 else np.mean(d.astype(np.float64))
    return out


def surface_dice(y_pred, y, class_thresholds, include_background=False, spacing=None) -> np.ndarray:
    y_pred, y = _drop_bg(y_pred, include_background), _drop_bg(y, include_background)
    b, c = y_pred.shape[:2]
    sp = _spacing_list(spacing, b)
    out = np.empty((b, c), np.float32)
    for i in range(b):
        for j in range(c):
            d0, d1 = (torch.from_numpy(d) for d in pair_distances(y_pred[i, j], y[i, j], sp[i]))
            complete = len(d0) + len(d1)
            if complete == 0:
                out[i, j] = np.nan
            else:
                correct = torch.sum(d0 <= class_thresholds[j]) + torch.sum(d1 <= class_thresholds[j])
                out[i, j] = (correct / complete).item()
    return out


def brute_force_distances(pred, gt, spacing=(1.0, 1.0, 1.0)):
    """the same two distance arrays by loops over every voxel and every edge voxel: for checking the oracle on tiny volumes"""
    def brute_edges(m):
        m = np.asarray(m, bool)
        e = np.zeros_like(m)
        D, H, W = m.shape
        for z, yy, x in zip(*np.nonzero(m)):
            for dz, dy, dx in ((-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)):
                a, b_, c_ = z + dz, yy + dy, x + dx
                if not (0 <= a < D and 0 <= b_ < H and 0 <= c_ < W) or not m[a, b_, c_]:
                    e[z, yy, x] = True
                    break
        return e

    s = [float(v) for v in spacing]
    ep, eg = brute_edges(foreground(pred)), brute_edges(foreground(gt))

    def one(eq, ef):
        if not ef.any():
            return np.full(int(eq.sum()), np.inf, np.float32)
        if not eq.any():
            return np.full(int(ef.sum()), np.inf, np.float32)
        fs = np.argwhere(ef)
        out = []
        for q in np.argwhere(eq):
            best = np.inf
            for f in fs:
                a, b_, c_ = ((f - q) * np.asarray(s)).tolist()
                best = min(best, np.sqrt((a * a + b_ * b_) + c_ * c_))
            out.append(best)
        return np.asarray(out, np.float64).astype(np.float32)

    return [one(ep, eg), one(eg, ep)]
