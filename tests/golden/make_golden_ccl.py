"""Masks and expected connected components for tests/golden/ccl.npz.

Every mask comes from a seed through integer arithmetic only (numpy PCG64 integer draws, integer sphere and box tests), so
``make_masks()`` regenerates them bit for bit without scipy: the GPU tests rebuild the masks here and compare the kernels with the
stored results.  The results come from tests/ccl_oracle.py (scipy.ndimage.label).  For every case and connectivity 1, 2, 3 the
fixture stores K, the sizes in size order and the SHA-256 of both numberings (int32, C order); the label arrays themselves only
for cases of at most 32^3 voxels.

    python tests/golden/make_golden_ccl.py      # writes tests/golden/ccl.npz
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
FULL_ARRAYS_MAX = 32 ** 3
CONNECTIVITIES = (1, 2, 3)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype="<i4").tobytes()).hexdigest()


def _rng(seed):
    return np.random.Generator(np.random.PCG64(seed))


def _grid(shape):
    return np.ogrid[:shape[0], :shape[1], :shape[2]]


def noise(shape, percent, seed):
    return (_rng(seed).integers(0, 100, size=shape, dtype=np.int64) < percent).astype(np.uint8)


def spheres(shape, n, rmin, rmax, seed):
    """union of n balls with integer centres and radii: dz^2 + dy^2 + dx^2 <= r^2"""
    rng = _rng(seed)
    z, y, x = _grid(shape)
    m = np.zeros(shape, np.uint8)
    for _ in range(n):
        c = [int(rng.integers(0, s)) for s in shape]
        r = int(rng.integers(rmin, rmax + 1))
        m |= ((z - c[0]) ** 2 + (y - c[1]) ** 2 + (x - c[2]) ** 2 <= r * r).astype(np.uint8)
    return m


def shell(shape=(40, 40, 40)):
    """a ball of radius 6 inside a hollow shell 10 <= r <= 13: two components, the shell the larger"""
    z, y, x = _grid(shape)
    r2 = (z - 20) ** 2 + (y - 19) ** 2 + (x - 21) ** 2
    return ((r2 <= 36) | ((r2 >= 100) & (r2 <= 169))).astype(np.uint8)


def cubes(shape=(32, 32, 32)):
    """4^3 boxes of sides 3, 4, 2, 3, ... at a pitch of 7: most are 27-voxel ties, so the size order is not the raster order"""
    m = np.zeros(shape, np.uint8)
    starts = (1, 8, 15, 22)
    for a, z0 in enumerate(starts):
        for b, y0 in enumerate(starts):
            for c, x0 in enumerate(starts):
                s = (3, 4, 2, 3)[(a + 2 * b + c) % 4]
                m[z0:z0 + s, y0:y0 + s, x0:x0 + s] = 1
    return m


def checker(shape):
    z, y, x = _grid(shape)
    return ((z + y + x) % 2 == 0).astype(np.uint8)


def corners(shape=(9, 10, 11)):
    m = np.zeros(shape, np.uint8)
    for z in (0, shape[0] - 1):
        for y in (0, shape[1] - 1):
            for x in (0, shape[2] - 1):
                m[z, y, x] = 1
    return m


def pair(offset, shape=(5, 5, 5)):
    m = np.zeros(shape, np.uint8)
    m[2, 2, 2] = 1
    m[2 + offset[0], 2 + offset[1], 2 + offset[2]] = 1
    return m


def tile_diagonals(shape=(12, 20, 70)):
    """pairs of voxels that touch only across the borders of 4 x 8 x 32 tiles: through a face, an edge or a corner, each
    pair far from the others"""
    m = np.zeros(shape, np.uint8)
    for a, b in [((3, 7, 31), (4, 8, 32)),      # corner: three tile borders at once
                 ((3, 2, 10), (4, 1, 10)),      # edge across a z border (dz = 1, dy = -1)
                 ((9, 7, 50), (9, 8, 51)),      # edge across a y and an x border
                 ((6, 15, 63), (7, 16, 64)),    # corner again, deeper
                 ((1, 12, 31), (1, 12, 32)),    # face across an x border
                 ((7, 4, 5), (8, 5, 4))]:       # corner with dx = -1
        m[a] = 1
        m[b] = 1
    return m


def serpentine(shape=(96, 80, 72)):
    """one voxel wide path through the whole volume: in every even slice the rows y = 0, 2, 4, ... joined at alternating ends
    through the odd rows; consecutive slices run the same path in opposite directions, joined at its ends through the odd
    slices.  Rows and slices are 2 apart, so the path touches itself nowhere, not even diagonally: one component at every
    connectivity, and the longest union chains, crossing every tile border."""
    D, H, W = shape
    m = np.zeros(shape, np.uint8)
    rows = list(range(0, H, 2))
    plane = np.zeros((H, W), np.uint8)
    end = None
    for r, y in enumerate(rows):
        plane[y, :] = 1
        end = (y, W - 1) if r % 2 == 0 else (y, 0)
        if r + 1 < len(rows):
            plane[y + 1, end[1]] = 1
    m[0::2] = plane
    for s, z in enumerate(range(1, D - 1, 2)):
        m[z][end if s % 2 == 0 else (0, 0)] = 1
    return m


def keep_largest_field(shape=(24, 20, 28), seed=808):
    """label field 0..3 for the keep-largest tests: balls of labels 1..3 (later ones overwrite) and single-voxel specks"""
    rng = _rng(seed)
    z, y, x = _grid(shape)
    q = np.zeros(shape, np.int64)
    for _ in range(9):
        c = [int(rng.integers(0, s)) for s in shape]
        r = int(rng.integers(2, 7))
        q[(z - c[0]) ** 2 + (y - c[1]) ** 2 + (x - c[2]) ** 2 <= r * r] = int(rng.integers(1, 4))
    for _ in range(30):
        q[tuple(int(rng.integers(0, s)) for s in shape)] = int(rng.integers(1, 4))
    return q


def make_masks():
    """name -> uint8 mask (D, H, W), in a fixed order"""
    m = {}
    m["empty_8x9x10"] = np.zeros((8, 9, 10), np.uint8)
    for shp in ((1, 1, 1), (1, 1, 300), (37, 41, 53)):
        m["full_%dx%dx%d" % shp] = np.ones(shp, np.uint8)
    m["corners_9x10x11"] = corners()
    m["pair_face"] = pair((0, 0, 1))
    m["pair_edge"] = pair((0, 1, 1))
    m["pair_corner"] = pair((1, 1, 1))
    m["tile_diagonals_12x20x70"] = tile_diagonals()
    m["checker_16x16x16"] = checker((16, 16, 16))
    m["checker_37x41x53"] = checker((37, 41, 53))
    m["serpentine_96x80x72"] = serpentine()
    m["shell_40x40x40"] = shell()
    m["cubes_32x32x32"] = cubes()
    m["spheres_64x64x64"] = spheres((64, 64, 64), 14, 3, 12, seed=11)
    m["spheres_96x80x72"] = spheres((96, 80, 72), 20, 2, 14, seed=12)
    m["noise50_1x1x1"] = noise((1, 1, 1), 50, seed=20)
    m["noise50_1x1x300"] = noise((1, 1, 300), 50, seed=21)
    for pct, seed in ((10, 30), (25, 31), (31, 32), (50, 33)):
        m["noise%d_37x41x53" % pct] = noise((37, 41, 53), pct, seed)
    m["noise25_32x32x32"] = noise((32, 32, 32), 25, seed=34)
    m["noise25_64x64x64"] = noise((64, 64, 64), 25, seed=35)
    m["noise31_96x80x72"] = noise((96, 80, 72), 31, seed=36)
    q = keep_largest_field()
    for name, vals in (("kl_l1", (1,)), ("kl_l2", (2,)), ("kl_l3", (3,)), ("kl_u13", (1, 3)), ("kl_u123", (1, 2, 3))):
        m[name] = np.isin(q, vals).astype(np.uint8)
    return m


# three different volumes of one shape, labelled in one batched call
BATCH = ("noise10_37x41x53", "noise31_37x41x53", "checker_37x41x53")


def main():
    sys.path.insert(0, os.path.dirname(HERE))
    from ccl_oracle import label_raster, size_order
    out = {}
    for name, mask in make_masks().items():
        out["%s__mask_sha" % name] = np.array(sha(mask))
        for conn in CONNECTIVITIES:
            raster, k = label_raster(mask, conn)
            bysize, sizes = size_order(raster, k)
            key = "%s__%d__" % (name, conn)
            out[key + "K"] = np.array(k, np.int64)
            out[key + "sizes"] = sizes.astype(np.int32)
            out[key + "sha_raster"] = np.array(sha(raster))
            out[key + "sha_size"] = np.array(sha(bysize))
            if mask.size <= FULL_ARRAYS_MAX:
                out[key + "raster"] = raster
                out[key + "bysize"] = bysize
        print("%-26s %s K(1,2,3) = %s" % (name, "x".join(map(str, mask.shape)),
                                         [int(out["%s__%d__K" % (name, c)]) for c in CONNECTIVITIES]))
    np.savez_compressed(os.path.join(HERE, "ccl.npz"), **out)


if __name__ == "__main__":
    main()
