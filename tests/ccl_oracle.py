"""Connected components restated on the host, for the tests and the fixture generator (test infrastructure only).

  * ``label_raster``: ``scipy.ndimage.label`` with ``generate_binary_structure(3, connectivity)``: labels 1..K in raster order
    of each component's first voxel.  Pinned to scipy (the fixture tests/golden/ccl.npz was written with scipy 1.18).
  * ``size_order``: renumbering by decreasing size, equal sizes in raster order (a stable sort).  This is the comparator of
    SimpleITK's ``RelabelComponent(sortByObjectSize=True)`` as its documentation states it; unpinned, SimpleITK is not installed.
  * ``keep_largest``: ``monai.transforms.KeepLargestConnectedComponent`` restated from MONAI's documentation and source, with
    the tie rule above at the ``num_components`` cut (MONAI's own ``argsort`` is unstable there); unpinned, MONAI is not
    installed.  The labeller is a parameter, so a caller without scipy can label from stored arrays.

scipy is imported on first use only: the GPU tests import this module without it.

It sits under tests/ beside dice_ce_oracle.py, the other test-only restatement, and not in the ``oracle`` package.  That
package holds the restatements of the reference model that build() imports and smoke() checks against; scipy is not among its
dependencies.
"""
import numpy as np


def label_raster(mask, connectivity):
    """mask (D, H, W), nonzero = foreground -> (int32 labels in raster order, K)"""
    from scipy import ndimage
    lab, k = ndimage.label(np.asarray(mask) != 0, structure=ndimage.generate_binary_structure(3, connectivity))
    return lab.astype(np.int32), int(k)


def size_order(raster, k):
    """raster labels 1..k -> (labels numbered by decreasing size with ties in raster order, sizes in that order)"""
    sizes = np.bincount(raster.ravel(), minlength=k + 1)[1:]
    order = np.argsort(-sizes, kind="stable")              # order[new - 1] = old - 1
    newlab = np.zeros(k + 1, np.int32)
    newlab[order + 1] = np.arange(1, k + 1, dtype=np.int32)
    return newlab[raster], sizes[order].astype(np.int64)


def sized_labels(mask, connectivity):
    lab, k = label_raster(mask, connectivity)
    return size_order(lab, k)[0]


def keep_largest(img, applied_labels=None, is_onehot=None, independent=True, connectivity=None, num_components=1,
                 labeller=sized_labels):
    """img: channel-first numpy array (C, D, H, W).  labeller(mask, connectivity) -> size-ordered labels of a boolean mask."""
    img = np.asarray(img)
    conn = 3 if connectivity is None else connectivity
    onehot = img.shape[0] > 1 if is_onehot is None else is_onehot
    if applied_labels is None:
        if onehot:
            applied = [i for i in range(img.shape[0]) if img[i].sum() > 0 and i != 0]
        else:
            applied = [v for v in np.unique(img).tolist() if v != 0]
    else:
        applied = list(applied_labels) if isinstance(applied_labels, (list, tuple)) else [applied_labels]
    out = img.copy()

    def keep(fg):
        return fg & (labeller(fg, conn) <= num_components)

    if independent:
        for i in applied:
            fg = img[i] > 0 if onehot else img[0] == i
            if onehot:
                out[i][fg != keep(fg)] = 0
            else:
                out[0][fg != keep(fg)] = 0
        return out
    if onehot:
        fg = (img[applied] == 1).any(0)
        k = keep(fg)
        for i in applied:
            out[i][fg != k] = 0
        return out
    fg = np.isin(img[0], applied)
    out[0][fg != keep(fg)] = 0
    return out
