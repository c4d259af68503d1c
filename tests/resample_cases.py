"""Grids and fp64 oracles for the resample of a prediction onto its image file's grid (``prepost.resample_to_match``).

A dataset transform that changes the grid maps each new voxel index to an old one, ``old = P @ new`` (4x4, homogeneous), so
the new affine is ``A @ P``; the helpers below build P for the transforms the training configs chain (orientation, foreground
crop, resize) the way MONAI updates the affine, and compose them from a file's affine."""
from fractions import Fraction

import numpy as np
from scipy import ndimage


def file_affine(spacing, origin=(0.0, 0.0, 0.0), lps=False):
    """voxel-to-world affine of a file with this voxel spacing; lps: the first two axes point to -x and -y (DICOM order)"""
    a = np.diag([float(s) for s in spacing] + [1.0])
    if lps:
        a[0, 0], a[1, 1] = -a[0, 0], -a[1, 1]
    a[:3, 3] = origin
    return a


def flip_perm(shape, perm=(0, 1, 2), flips=()):
    """new axis i reads old axis perm[i], reversed when i is in flips (an Orientation to another axis code).  Returns
    (P, new shape)."""
    p = np.zeros((4, 4))
    p[3, 3] = 1.0
    for i, j in enumerate(perm):
        if i in flips:
            p[j, i], p[j, 3] = -1.0, shape[j] - 1.0
        else:
            p[j, i] = 1.0
    return p, tuple(shape[j] for j in perm)


def crop(start):
    """foreground crop starting at old index ``start``: old = new + start"""
    p = np.eye(4)
    p[:3, 3] = start
    return p


def resize(old_shape, new_shape):
    """Resize (align_corners=False): old = (new + 0.5) * old / new - 0.5"""
    s = np.asarray(old_shape, dtype=np.float64) / np.asarray(new_shape, dtype=np.float64)
    p = np.diag(list(s) + [1.0])
    p[:3, 3] = (s - 1) / 2
    return p


def unflip_perm(shape, perm=(0, 1, 2), flips=()):
    """the inverse of flip_perm, written out: new_i = old_perm[i], or shape[perm[i]] - 1 - old_perm[i] when i is in flips"""
    q = np.zeros((4, 4))
    q[3, 3] = 1.0
    for i, j in enumerate(perm):
        if i in flips:
            q[i, j], q[i, 3] = -1.0, shape[j] - 1.0
        else:
            q[i, j] = 1.0
    return q


def unresize(old_shape, new_shape):
    """the inverse of resize, written out: new = (old + 0.5) * new / old - 0.5"""
    s = np.asarray(new_shape, dtype=np.float64) / np.asarray(old_shape, dtype=np.float64)
    q = np.diag(list(s) + [1.0])
    q[:3, 3] = (s - 1) / 2
    return q


# file grid and the dataset's steps: orientation (axis permutation + flips), foreground crop [start, start + box), resize
GRIDS = {
    # a 240 x 240 x 155 LPS file at 1 mm oriented to RAS and resized to 128^3, as the BraTS config does
    "brats": dict(spacing=(1.0, 1.0, 1.0), origin=(0.0, 239.0, 0.0), lps=True, angle=0.0, shape=(240, 240, 155), perm=(0, 1, 2),
                  flips=(0, 1), start=(30, 25, 10), box=(180, 195, 140), out=(128, 128, 128)),
    # an anisotropic 256 x 256 x 160 file (0.7 x 0.7 x 1.2 mm) stored (h, w, d) under an oblique, non-diagonal affine, resized
    # to 192^3 as the SPPIN config does
    "sppin": dict(spacing=(0.7, 0.7, 1.2), origin=(-90.0, 80.0, -40.0), lps=False, angle=0.3, shape=(256, 256, 160), perm=(2, 0, 1),
                  flips=(1,), start=(8, 20, 16), box=(144, 216, 224), out=(192, 192, 192)),
}


def grid(name):
    """(file affine, file shape, prediction affine, prediction shape)"""
    g = GRIDS[name]
    c, s = np.cos(g["angle"]), np.sin(g["angle"])
    rot = np.array([[c, -s, 0, 0], [s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1.0]])
    a0 = rot @ file_affine(g["spacing"], g["origin"], g["lps"])
    po, oshape = flip_perm(g["shape"], g["perm"], g["flips"])
    assert all(st + b <= n for st, b, n in zip(g["start"], g["box"], oshape))
    return a0, g["shape"], a0 @ po @ crop(g["start"]) @ resize(g["box"], g["out"]), g["out"]


def expected_index_map(name):
    """file index -> prediction index from the steps' inverses, written out: unresize @ uncrop @ unorient"""
    g = GRIDS[name]
    return (unresize(g["box"], g["out"]) @ crop(-np.asarray(g["start"], dtype=np.float64))
            @ unflip_perm(g["shape"], g["perm"], g["flips"]))[:3]


def target_coords(m, dst_shape):
    """fp64 source index of every target voxel: [3, *dst_shape]"""
    g = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in dst_shape], indexing="ij")
    return np.stack([m[i, 0] * g[0] + m[i, 1] * g[1] + m[i, 2] * g[2] + m[i, 3] for i in range(3)])


def _fma(a, b, c):
    """fp64 fused multiply-add, rounded once (exact rational arithmetic, then round to nearest even)"""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def _tie_exact(m, x, band=1e-9):
    """where a coordinate lies within ``band`` of a rounding tie, recompute it as the kernel does: fma(m0, d, fma(m1, h,
    fma(m2, w, m3))), each fma rounded once.  Separately rounded products can land on the other side of a tie
    (1.2 * 2 + 1.1 gives 3.5 in numpy, 3.4999999999999996 fused), and nearest mode is compared exactly."""
    near = np.abs(x - np.floor(x) - 0.5) < band
    for i, d, h, w in zip(*np.nonzero(near)):
        r = [float(v) for v in m[i]]
        x[i, d, h, w] = _fma(r[0], float(d), _fma(r[1], float(h), _fma(r[2], float(w), r[3])))
    return x


def oracle(vol, m, dst_shape, mode="trilinear"):
    """fp64 resample of vol [C, D, H, W] through the 3x4 index map m with border padding: trilinear is
    scipy.ndimage.map_coordinates(order=1, mode="nearest"); nearest clamps and rounds half to even"""
    vol = np.asarray(vol, dtype=np.float64)
    x = target_coords(m, dst_shape)
    if mode == "nearest":
        x = _tie_exact(m, x)
        idx = [np.rint(np.clip(x[i], 0, vol.shape[1 + i] - 1)).astype(np.int64) for i in range(3)]
        return np.stack([v[idx[0], idx[1], idx[2]] for v in vol])
    return np.stack([ndimage.map_coordinates(v, x, order=1, mode="nearest") for v in vol])
