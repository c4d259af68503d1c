"""Connected components on the GPU: both numberings bit-exact against every case of tests/golden/ccl.npz at every connectivity
(masks regenerated from their seeds, no scipy), a batched call, 256^3 blobs and noise against a torch restatement run here,
the keep-largest matrix against expectations derived from the stored label arrays, and run-to-run equality."""
import functools
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import ccl_oracle as oracle  # noqa: E402
from make_golden_ccl import BATCH, CONNECTIVITIES, FULL_ARRAYS_MAX, keep_largest_field, make_masks, sha, spheres  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = np.load(os.path.join(HERE, "golden", "ccl.npz"))
MASKS = make_masks()


def _raster(pkg, m, conn):
    """the labelling call alone: raster-order labels and counts of m [nvol, d, h, w] uint8"""
    L = pkg.lib
    nvol, d, h, w = m.shape
    labels = torch.empty(m.shape, dtype=torch.int32, device=m.device)
    counts = torch.empty(nvol, dtype=torch.int32, device=m.device)
    scratch = torch.empty(L.cc_scratch_bytes(nvol, d, h, w), dtype=torch.uint8, device=m.device)
    L.cc_label(m.contiguous(), conn, labels, counts, scratch)
    return labels, counts


def _expect(name, conn, raster, bysize, count):
    key = "%s__%d__" % (name, conn)
    assert count == int(GOLD[key + "K"]), (name, conn, count)
    if MASKS[name].size <= FULL_ARRAYS_MAX:
        assert np.array_equal(raster, GOLD[key + "raster"]), (name, conn)
        assert np.array_equal(bysize, GOLD[key + "bysize"]), (name, conn)
    assert sha(raster) == str(GOLD[key + "sha_raster"]), (name, conn)
    assert sha(bysize) == str(GOLD[key + "sha_size"]), (name, conn)
    sizes = np.bincount(bysize.ravel(), minlength=count + 1)[1:]
    assert np.array_equal(sizes, GOLD[key + "sizes"])


@pytest.mark.parametrize("conn", CONNECTIVITIES)
@pytest.mark.parametrize("name", sorted(MASKS))
def test_both_numberings_match_the_fixture(pkg, name, conn):
    m = torch.from_numpy(MASKS[name]).to(DEV)
    raster, counts = _raster(pkg, m[None], conn)
    bysize, k = pkg.prepost.connected_components(m, connectivity=conn)
    assert k.dtype == torch.int64 and k.shape == () and int(counts[0]) == int(k)
    assert bysize.dtype == torch.int32 and bysize.shape == m.shape
    _expect(name, conn, raster[0].cpu().numpy(), bysize.cpu().numpy(), int(k))


@pytest.mark.parametrize("conn", CONNECTIVITIES)
def test_batch_of_three_volumes(pkg, conn):
    m = torch.stack([torch.from_numpy(MASKS[n]) for n in BATCH]).to(DEV)
    raster, counts = _raster(pkg, m, conn)
    bysize, k = pkg.prepost.connected_components(m.bool().view(3, 1, *m.shape[1:]), connectivity=conn)
    assert k.shape == (3, 1) and bysize.shape == (3, 1) + tuple(m.shape[1:])
    for i, name in enumerate(BATCH):
        assert int(counts[i]) == int(k[i, 0])
        _expect(name, conn, raster[i].cpu().numpy(), bysize[i, 0].cpu().numpy(), int(k[i, 0]))


# ------------------------------------------------------------------------------------------------ 256^3 against torch
BACK = [(-1, 0, 0), (0, -1, 0), (0, 0, -1), (-1, -1, 0), (-1, 1, 0), (-1, 0, -1), (-1, 0, 1), (0, -1, -1), (0, -1, 1),
        (-1, -1, -1), (-1, -1, 1), (-1, 1, -1), (-1, 1, 1)]


def _pair_slices(shape, off):
    """views a, b of a volume such that b[p] is the neighbour of a[p] at offset off"""
    sa, sb = [], []
    for n, o in zip(shape, off):
        sa.append(slice(max(0, -o), n - max(0, o)))
        sb.append(slice(max(0, o), n - max(0, -o)))
    return tuple(sa), tuple(sb)


def torch_components(m, conn, cap=3000):
    """Independent restatement: min-label propagation over the neighbour pairs plus pointer jumping, to the fixed point where
    every voxel holds the minimum linear index of its component; raster labels by a prefix sum over those roots, size order
    by a stable sort.  Fails the test when the cap is hit."""
    D, H, W = m.shape
    S = m.numel()
    idx = torch.arange(S, device=m.device, dtype=torch.int64).view(D, H, W)
    big = torch.full_like(idx, S)
    lab = torch.where(m, idx, big)
    pairs = [_pair_slices(m.shape, off) for off in BACK[:{1: 3, 2: 9, 3: 13}[conn]]]
    pairs = [(sa, sb, m[sa] & m[sb]) for sa, sb in pairs]
    flat = lab.view(-1)
    for _ in range(cap):
        prev = lab.clone()
        for sa, sb, both in pairs:
            mn = torch.where(both, torch.minimum(lab[sa], lab[sb]), S)
            lab[sa] = torch.minimum(lab[sa], mn)        # the two views overlap: each write only lowers what is there
            lab[sb] = torch.minimum(lab[sb], mn)
        while True:
            jumped = torch.where(m.view(-1), flat[flat.clamp(max=S - 1)], flat)
            if torch.equal(jumped, flat):
                break
            flat.copy_(jumped)
        if torch.equal(lab, prev):
            break
    else:
        pytest.fail("torch restatement did not converge in %d rounds" % cap)
    roots = (lab == idx) & m
    rank = torch.cumsum(roots.view(-1).to(torch.int64), 0)
    raster = torch.where(m.view(-1), rank[flat.clamp(max=S - 1)], 0).view(D, H, W)
    k = int(rank[-1])
    sizes = torch.bincount(raster.view(-1), minlength=k + 1)[1:]
    order = torch.sort(sizes, descending=True, stable=True).indices
    newlab = torch.zeros(k + 1, dtype=torch.int64, device=m.device)
    newlab[order + 1] = torch.arange(1, k + 1, device=m.device)
    return raster, newlab[raster], k


@functools.lru_cache(maxsize=None)
def _blobs_np(n, seed):
    return spheres((n, n, n), 40, 4, 30, seed)


def _blobs(n=256, seed=5):
    return torch.from_numpy(_blobs_np(n, seed)).to(DEV)


def _noise(n=256, seed=6, percent=25):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randint(0, 100, (n, n, n), device=DEV, generator=g) < percent).to(torch.uint8)


@pytest.mark.parametrize("conn", [1, 3])
@pytest.mark.parametrize("kind", ["blobs", "noise25"])
def test_256_cubed_matches_torch_restatement(pkg, kind, conn):
    m = _blobs() if kind == "blobs" else _noise()
    raster, counts = _raster(pkg, m[None], conn)
    bysize, k = pkg.prepost.connected_components(m, connectivity=conn)
    t_raster, t_bysize, tk = torch_components(m.bool(), conn)
    assert int(counts[0]) == int(k) == tk
    assert tk > (1 if kind == "blobs" else 1000)
    assert torch.equal(raster[0].long(), t_raster)
    assert torch.equal(bysize.long(), t_bysize)


def test_repeats_are_identical_at_256_cubed(pkg):
    m = torch.stack([_noise(seed=7, percent=31), _blobs(seed=8)])
    for conn in (1, 3):
        first = pkg.prepost.connected_components(m, connectivity=conn)
        for _ in range(2):
            again = pkg.prepost.connected_components(m, connectivity=conn)
            assert torch.equal(again[0], first[0]) and torch.equal(again[1], first[1])


# ------------------------------------------------------------------------------------------------ keep largest
KL_NAMES = ("kl_l1", "kl_l2", "kl_l3", "kl_u13", "kl_u123")
BY_SHA = {str(GOLD["%s__mask_sha" % n]): n for n in KL_NAMES}


def stored_labeller(fg, conn):
    """size-ordered labels of a keep-largest mask, from the fixture (each mask the matrix builds is one of KL_NAMES)"""
    return GOLD["%s__%d__bysize" % (BY_SHA[sha(fg)], conn)]


NP = {torch.uint8: np.uint8, torch.int16: np.int16, torch.int64: np.int64, torch.float32: np.float32}


@pytest.mark.parametrize("dtype", list(NP))
@pytest.mark.parametrize("form", ["label_map", "one_hot"])
def test_keep_largest_matrix(pkg, form, dtype):
    q = keep_largest_field()
    img_np = (q[None] if form == "label_map" else np.stack([q == c for c in range(4)])).astype(NP[dtype])
    img = torch.from_numpy(img_np).to(DEV)
    before = img.clone()
    checked = 0
    for independent in (True, False):
        for applied in (None, [1, 3], [2]):
            for n in (1, 2):
                for conn in (None, 1):
                    kw = dict(applied_labels=applied, independent=independent, connectivity=conn, num_components=n)
                    got = pkg.prepost.keep_largest_connected_component(img, **kw)
                    exp = oracle.keep_largest(img_np, labeller=stored_labeller, **kw)
                    assert got.dtype == dtype and got.shape == img.shape
                    assert np.array_equal(got.cpu().numpy(), exp), kw
                    assert torch.equal(img, before)
                    checked += int(not np.array_equal(exp, img_np))
    assert checked >= 20                     # the matrix drops components in most of its 24 settings


def test_keep_largest_is_onehot_flag(pkg):
    """a one-channel image treated as one-hot cleans channel 0 (the applied label must be given: 0 is discarded otherwise)"""
    m = MASKS["kl_l3"]
    img = torch.from_numpy(m[None].astype(np.float32)).to(DEV)
    got = pkg.prepost.keep_largest_connected_component(img, applied_labels=[0], is_onehot=True, connectivity=1)
    exp = m * (GOLD["kl_l3__1__bysize"] == 1)
    assert np.array_equal(got[0].cpu().numpy(), exp.astype(np.float32))


@pytest.mark.parametrize("conn", [1, 3])
def test_strided_inputs_give_the_contiguous_result(pkg, conn):
    """Fortran-order (nibabel's NIfTI layout) and permuted float masks, and a permuted one-hot image, label exactly as their
    C-order copies"""
    name = "noise31_37x41x53"
    c_order = torch.from_numpy(MASKS[name].astype(np.float32)).to(DEV)
    fortran = torch.from_numpy(np.asfortranarray(MASKS[name].astype(np.float32))).to(DEV)
    permuted = c_order.permute(2, 1, 0).contiguous().permute(2, 1, 0)
    assert not fortran.is_contiguous() and not permuted.is_contiguous()
    ref, k = pkg.prepost.connected_components(c_order, connectivity=conn)
    _expect(name, conn, _raster(pkg, c_order.to(torch.uint8)[None], conn)[0][0].cpu().numpy(), ref.cpu().numpy(), int(k))
    for m in (fortran, permuted):
        got, kk = pkg.prepost.connected_components(m, connectivity=conn)
        assert int(kk) == int(k) and torch.equal(got, ref)
    q = torch.from_numpy(keep_largest_field()).to(DEV)
    onehot = torch.stack([q == c for c in range(4)]).to(torch.float32)
    strided = onehot.permute(0, 3, 2, 1).contiguous().permute(0, 3, 2, 1)
    assert not strided.is_contiguous()
    for kw in (dict(), dict(independent=False, applied_labels=[1, 3])):
        want = pkg.prepost.keep_largest_connected_component(onehot, connectivity=conn, **kw)
        got = pkg.prepost.keep_largest_connected_component(strided, connectivity=conn, **kw)
        assert not torch.equal(want, onehot) and torch.equal(got, want)
