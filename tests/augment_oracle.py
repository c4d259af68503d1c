"""fp64 CPU restatement of ``augment.Compose`` for one batch, from the parameters it drew (``Compose.last_params``):
resample with ``F.grid_sample(align_corners=False)`` on the composed index-space affine converted to normalised coordinates
(trilinear image, nearest label), then z-score and the composed scale / shift.  Independent of csrc/augment.cu."""
import torch
import torch.nn.functional as F


def source_coordinates(affine: torch.Tensor, spatial) -> torch.Tensor:
    """affine fp64 [N][3][4] -> source index (d, h, w) of every output voxel, fp64 [N][D][H][W][3]."""
    d, h, w = spatial
    grid = torch.stack(torch.meshgrid(torch.arange(d, dtype=torch.float64), torch.arange(h, dtype=torch.float64),
                                      torch.arange(w, dtype=torch.float64), indexing="ij"), dim=-1)
    a = affine.to(torch.float64)
    return torch.einsum("nij,dhwj->ndhwi", a[:, :, :3], grid) + a[:, None, None, None, :, 3]


def resample(x: torch.Tensor, affine: torch.Tensor, padding_mode: str, mode: str) -> torch.Tensor:
    """x [N][C][D][H][W] (any dtype) -> fp64 resampled at source_coordinates; mode "bilinear" (trilinear) or "nearest"."""
    spatial = tuple(x.shape[2:])
    src = source_coordinates(affine, spatial)
    size = torch.tensor(spatial, dtype=torch.float64)
    norm = (2.0 * src + 1.0) / size - 1.0                    # align_corners=False: index i <-> (2i + 1) / size - 1
    grid = norm.flip(-1)                                      # grid_sample wants (x, y, z) = (w, h, d)
    return F.grid_sample(x.to(torch.float64), grid, mode=mode, padding_mode=padding_mode, align_corners=False)


def intensity(y: torch.Tensor, normalize, coef: torch.Tensor) -> torch.Tensor:
    """z-score (population std, std 0 -> 1; nonzero: over and on the non-zero voxels) then y * a + b per (n, c), fp64."""
    y = y.clone()
    if normalize is not None:
        n, c = y.shape[:2]
        groups = [(i, [j]) for i in range(n) for j in range(c)] if normalize["channel_wise"] else [(i, list(range(c))) for i in range(n)]
        for i, chans in groups:
            v = y[i, chans]
            # grid_sample's round trip through normalised coordinates puts an integer source coordinate ~1e-15 off, so a
            # copied 0 can come out as ~1e-15 times its neighbour: count those as the zeros they are
            sel = v.abs() > 1e-12 if normalize["nonzero"] else torch.ones_like(v, dtype=torch.bool)
            if sel.any():
                m = v[sel].mean()
                s = v[sel].std(unbiased=False)
                s = s if s != 0 else torch.tensor(1.0, dtype=torch.float64)
                v = torch.where(sel, (v - m) / s, v)
            y[i, chans] = v
    coef = coef.to(torch.float64)
    return y * coef[:, :, 0, None, None, None] + coef[:, :, 1, None, None, None]


def augment(image: torch.Tensor, label, params: dict):
    """The batch ``Compose`` produced for ``params`` (its ``last_params``): fp64 image, fp64 label (or None)."""
    y = intensity(resample(image, params["affine"], params["padding_mode"], "bilinear"), params["normalize"], params["coef"])
    lab = None if label is None else resample(label, params["affine"], params["padding_mode"], "nearest")
    return y, lab
