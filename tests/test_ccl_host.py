"""Connected components without a GPU: the scipy oracle on hand-derived cases, the fixture masks regenerated from their seeds,
the marshalling of the three C-ABI calls against a recording stub, and the errors raised before any launch."""
import contextlib
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import ccl_oracle as oracle  # noqa: E402
from make_golden_ccl import BATCH, CONNECTIVITIES, FULL_ARRAYS_MAX, make_masks, sha  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "ccl.npz"))
MASKS = make_masks()


# ------------------------------------------------------------------------------------------------ the oracle, by hand
@pytest.mark.parametrize("name, expected", [
    ("pair_face", (1, 1, 1)),          # a shared face joins at every connectivity
    ("pair_edge", (2, 1, 1)),          # a shared edge needs 18 neighbours
    ("pair_corner", (2, 2, 1)),        # a shared corner needs 26
    ("corners_9x10x11", (8, 8, 8)),
    ("empty_8x9x10", (0, 0, 0)),
])
def test_oracle_counts_by_hand(name, expected):
    pytest.importorskip("scipy")
    assert tuple(oracle.label_raster(MASKS[name], c)[1] for c in CONNECTIVITIES) == expected


@pytest.mark.parametrize("shape", [(2, 2, 2), (3, 4, 5), (16, 16, 16)])
def test_oracle_checkerboard(shape):
    """6-connected, every voxel of a checkerboard is alone: ceil(S / 2) components of one voxel; through edges they all join"""
    pytest.importorskip("scipy")
    z, y, x = np.indices(shape)
    m = (z + y + x) % 2 == 0
    lab, k = oracle.label_raster(m, 1)
    assert k == (m.size + 1) // 2
    assert np.array_equal(lab[m], np.arange(1, k + 1))             # raster order of the first (only) voxel
    assert oracle.label_raster(m, 2)[1] == 1 and oracle.label_raster(m, 3)[1] == 1


def test_oracle_raster_and_size_order_by_hand():
    pytest.importorskip("scipy")
    m = np.zeros((1, 3, 9), np.uint8)
    m[0, 0, 0] = 1                          # A: size 1, first in raster order
    m[0, 0, 2:4] = 1                        # B: size 2
    m[0, 0, 6] = 1                          # C: size 1
    m[0, 2, 0:2] = 1                        # D: size 2, after B in raster order
    m[0, 2, 4:8] = 1                        # E: size 4
    lab, k = oracle.label_raster(m, 1)
    assert k == 5
    assert [lab[0, 0, 0], lab[0, 0, 2], lab[0, 0, 6], lab[0, 2, 0], lab[0, 2, 4]] == [1, 2, 3, 4, 5]
    bysize, sizes = oracle.size_order(lab, k)
    assert sizes.tolist() == [4, 2, 2, 1, 1]
    # E first; the ties keep raster order: B before D, A before C
    assert [bysize[0, 2, 4], bysize[0, 0, 2], bysize[0, 2, 0], bysize[0, 0, 0], bysize[0, 0, 6]] == [1, 2, 3, 4, 5]


def test_oracle_keep_largest_by_hand():
    pytest.importorskip("scipy")
    img = np.zeros((1, 1, 3, 9), np.int64)
    img[0, 0, 0, 0:2] = 1                   # label 1: sizes 2, 2 (a tie) and 3
    img[0, 0, 0, 4:6] = 1
    img[0, 0, 2, 0:3] = 1
    img[0, 0, 2, 3:7] = 2                   # label 2: one component of 4, touching label 1's largest through a face
    out = oracle.keep_largest(img)
    assert out[0, 0, 0].sum() == 0 and np.array_equal(out[0, 0, 2], img[0, 0, 2])
    out2 = oracle.keep_largest(img, num_components=2)
    assert out2[0, 0, 0, 0:2].tolist() == [1, 1] and out2[0, 0, 0, 4:6].tolist() == [0, 0]   # the tie goes to raster order
    assert np.array_equal(out2[0, 0, 2], img[0, 0, 2])
    union = oracle.keep_largest(img, independent=False)            # one component of 7, two of 2
    assert np.array_equal(union, out)
    only2 = oracle.keep_largest(img, applied_labels=[2], independent=False)
    assert np.array_equal(only2, img)
    onehot = np.stack([img[0] == 0, img[0] == 1, img[0] == 2]).astype(np.uint8)
    oh = oracle.keep_largest(onehot)                               # channel 0 is background: untouched
    assert np.array_equal(oh[0], onehot[0]) and np.array_equal(oh[1], (out[0] == 1).astype(np.uint8))
    assert np.array_equal(oh[2], onehot[2])


# ------------------------------------------------------------------------------------------------ the fixture
def test_fixture_masks_regenerate_from_their_seeds():
    names = {k.split("__")[0] for k in GOLD.files}
    assert names == set(MASKS)
    for name, m in MASKS.items():
        assert m.dtype == np.uint8
        assert sha(m) == str(GOLD["%s__mask_sha" % name]), name
    assert len({MASKS[n].shape for n in BATCH}) == 1


def test_fixture_stored_results_are_consistent():
    for name, m in MASKS.items():
        for conn in CONNECTIVITIES:
            key = "%s__%d__" % (name, conn)
            sizes = GOLD[key + "sizes"]
            assert len(sizes) == int(GOLD[key + "K"]) and int(sizes.sum()) == int((m != 0).sum())
            assert (np.diff(sizes) <= 0).all()
            if m.size <= FULL_ARRAYS_MAX:
                raster, bysize = GOLD[key + "raster"], GOLD[key + "bysize"]
                assert sha(raster) == str(GOLD[key + "sha_raster"]) and sha(bysize) == str(GOLD[key + "sha_size"])
                assert np.array_equal(bysize, oracle.size_order(raster, len(sizes))[0])


@pytest.mark.parametrize("name", sorted(MASKS))
def test_fixture_matches_scipy(name):
    pytest.importorskip("scipy")
    for conn in CONNECTIVITIES:
        raster, k = oracle.label_raster(MASKS[name], conn)
        bysize, sizes = oracle.size_order(raster, k)
        key = "%s__%d__" % (name, conn)
        assert k == int(GOLD[key + "K"]) and np.array_equal(sizes, GOLD[key + "sizes"])
        assert sha(raster) == str(GOLD[key + "sha_raster"]) and sha(bysize) == str(GOLD[key + "sha_size"])


# ------------------------------------------------------------------------------------------------ errors before any launch
@pytest.fixture()
def no_library(pkg, monkeypatch):
    def boom(*_a, **_k):
        raise AssertionError("the library was touched")
    monkeypatch.setattr(pkg.lib, "load_library", boom)
    monkeypatch.setattr(pkg.lib, "_lib", None)


def test_cpu_tensor_has_no_fallback(pkg, no_library):
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pkg.prepost.connected_components(torch.ones(4, 4, 4, dtype=torch.uint8))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pkg.prepost.keep_largest_connected_component(torch.ones(1, 4, 4, 4))


@pytest.mark.parametrize("conn", [0, 4, -1, 1.5, "1", True])
def test_bad_connectivity(pkg, no_library, conn):
    with pytest.raises(ValueError, match="connectivity"):
        pkg.prepost.connected_components(torch.ones(4, 4, 4, dtype=torch.uint8), connectivity=conn)
    with pytest.raises(ValueError, match="connectivity"):
        pkg.prepost.keep_largest_connected_component(torch.ones(1, 4, 4, 4), connectivity=conn)


# ------------------------------------------------------------------------------------------------ C-ABI marshalling
class _FakeCuda(torch.Tensor):
    is_cuda = True


SCRATCH = 4096


@pytest.fixture()
def recorded(pkg, monkeypatch):
    """every entry point of lib._SIGS replaced by a recorder that checks the argument count and types; cc_label writes
    counts = 1, 2, 3, ... (host memory stands in for the device) so the size sort receives a known maximum"""
    L = pkg.lib
    calls = []

    class Stub:
        pass
    stub = Stub()
    for name, (res, argtypes) in L._SIGS.items():
        def make(name=name, argtypes=argtypes):
            def f(*args):
                assert len(args) == len(argtypes), "%s: %d arguments, signature has %d" % (name, len(args), len(argtypes))
                for i, (v, t) in enumerate(zip(args, argtypes)):
                    try:
                        t.from_param(v)
                    except Exception as e:  # noqa: BLE001
                        raise AssertionError("%s: argument %d (%r) does not convert to %s: %s" % (name, i, v, t, e))
                calls.append((name, args))
                if name == "b200unet_cc_scratch_bytes":
                    return SCRATCH
                if name == "b200unet_cc_label":
                    nvol = args[1]
                    (C.c_int32 * nvol).from_address(args[7])[:] = list(range(1, nvol + 1))
                return 0
            return f
        setattr(stub, name, make())
    monkeypatch.setattr(L, "_lib", stub)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    monkeypatch.setattr(torch.cuda, "device", lambda *_a, **_k: contextlib.nullcontext())
    return calls


@pytest.mark.parametrize("dtype", [torch.uint8, torch.bool, torch.float32, torch.int64])
@pytest.mark.parametrize("conn", [1, 2, 3])
def test_connected_components_marshal(pkg, recorded, dtype, conn):
    mask = torch.zeros(2, 3, 5, 6, 7, dtype=dtype).as_subclass(_FakeCuda)
    labels, counts = pkg.prepost.connected_components(mask, connectivity=conn)
    names = [n for n, _ in recorded]
    assert names == ["b200unet_cc_scratch_bytes", "b200unet_cc_label", "b200unet_cc_sort_by_size"]
    assert recorded[0][1] == (6, 5, 6, 7)
    lab_args, sort_args = recorded[1][1], recorded[2][1]
    assert lab_args[1:6] == (6, 5, 6, 7, conn)
    assert lab_args[6] == labels.data_ptr() and sort_args[0] == labels.data_ptr()
    assert lab_args[8] == sort_args[6]                              # one scratch buffer serves both calls
    assert sort_args[1:6] == (6, 5, 6, 7, 6)                        # max_count = the largest of the counts read back
    assert labels.dtype == torch.int32 and labels.shape == mask.shape
    assert counts.dtype == torch.int64 and counts.device.type == "cpu" and counts.tolist() == [[1, 2, 3], [4, 5, 6]]


def test_keep_largest_marshals_one_batched_call(pkg, recorded):
    img = torch.zeros(4, 5, 6, 7, dtype=torch.int16).as_subclass(_FakeCuda)
    out = pkg.prepost.keep_largest_connected_component(img, connectivity=1)          # one-hot: channels 1..3, one call
    names = [n for n, _ in recorded]
    assert names == ["b200unet_cc_scratch_bytes", "b200unet_cc_label", "b200unet_cc_sort_by_size"]
    assert recorded[1][1][1:6] == (3, 5, 6, 7, 1)
    assert out.dtype == img.dtype and out.shape == img.shape and out.data_ptr() != img.data_ptr()
    recorded.clear()
    pkg.prepost.keep_largest_connected_component(img, independent=False, applied_labels=[1, 3])
    assert recorded[1][1][1:6] == (1, 5, 6, 7, 3)                                    # the union is one volume; None -> 26
    recorded.clear()
    lm = torch.zeros(1, 5, 6, 7, dtype=torch.float32).as_subclass(_FakeCuda)
    pkg.prepost.keep_largest_connected_component(lm, applied_labels=[1, 2, 5])
    assert recorded[1][1][1:6] == (3, 5, 6, 7, 3)


def test_keep_largest_without_labels_launches_nothing(pkg, recorded):
    lm = torch.zeros(1, 5, 6, 7, dtype=torch.uint8).as_subclass(_FakeCuda)          # a label map with no label but 0
    out = pkg.prepost.keep_largest_connected_component(lm)
    assert recorded == [] and out.shape == lm.shape


def test_bindings_refuse_non_contiguous_tensors(pkg, no_library):
    """the kernels read dense C-order [nvol, d, h, w] arrays: a strided view is refused before the library is touched"""
    m = torch.zeros(2, 4, 5, 6, dtype=torch.uint8)
    lab = torch.zeros(2, 4, 5, 6, dtype=torch.int32)
    with pytest.raises(ValueError, match="contiguous"):
        pkg.lib.cc_label(m.transpose(1, 3), 1, lab.transpose(1, 3), torch.zeros(2, dtype=torch.int32), torch.zeros(8))
    with pytest.raises(ValueError, match="contiguous"):
        pkg.lib.cc_label(m, 1, lab.transpose(1, 3), torch.zeros(2, dtype=torch.int32), torch.zeros(8))
    with pytest.raises(ValueError, match="contiguous"):
        pkg.lib.cc_sort_by_size(lab.transpose(1, 3), 3, torch.zeros(8))


@pytest.mark.parametrize("layout", ["fortran", "permuted"])
def test_strided_masks_reach_the_library_in_c_order(pkg, recorded, layout):
    """a Fortran-order array (as nibabel returns NIfTI data) or a permuted view keeps its strides through the mask predicate;
    the call must still see a C-order copy of the mask in the tensor's logical order"""
    seen = []
    orig = pkg.lib.cc_label

    def spy(mask, *a):
        seen.append((mask.is_contiguous(), mask.clone()))
        return orig(mask, *a)
    pkg.lib.cc_label, restore = spy, orig
    try:
        base = torch.arange(2 * 5 * 6 * 7, dtype=torch.float32).reshape(2, 5, 6, 7) % 3
        if layout == "fortran":
            pred = torch.from_numpy(np.asfortranarray(base.numpy()))
        else:
            pred = base.permute(0, 3, 2, 1).contiguous().permute(0, 3, 2, 1)
        assert not pred.is_contiguous() and torch.equal(pred, base)
        pkg.prepost.connected_components(pred.as_subclass(_FakeCuda), connectivity=1)
        onehot = torch.stack([base[0] == 0, base[0] == 1, base[0] == 2]).to(torch.int16).permute(0, 3, 2, 1).contiguous().permute(0, 3, 2, 1)
        assert not onehot.is_contiguous()
        pkg.prepost.keep_largest_connected_component(onehot.as_subclass(_FakeCuda))
    finally:
        pkg.lib.cc_label = restore
    assert [c for c, _ in seen] == [True, True]
    assert torch.equal(seen[0][1].as_subclass(torch.Tensor), (base != 0).to(torch.uint8))
    assert torch.equal(seen[1][1].as_subclass(torch.Tensor), torch.stack([base[0] == 1, base[0] == 2]).to(torch.uint8))


def test_keep_largest_empty_extent_launches_nothing(pkg, recorded):
    img = torch.zeros(3, 0, 6, 7, dtype=torch.float32).as_subclass(_FakeCuda)
    out = pkg.prepost.keep_largest_connected_component(img)
    assert recorded == [] and out.shape == img.shape and out.dtype == img.dtype
    lab, k = pkg.prepost.connected_components(torch.zeros(2, 4, 0, 5).as_subclass(_FakeCuda))
    assert recorded == [] and lab.shape == (2, 4, 0, 5) and k.tolist() == [0, 0]
