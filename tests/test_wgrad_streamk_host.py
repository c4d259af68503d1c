"""The stream-K partition of the per-tap weight gradient (wgrad.cu: wgrad_tiling, k_wgrad), restated in Python and held to the
library's route query over the weight-gradient launch shapes (tests/plan_launches.py) of the C2 and C3 UNet3D plans, the BraTS
DynUNet plan and the BraTS SegResNet recipe (batch 1 at 224 x 224 x 144, batch 2 at 128^3), on 114 and 132 SMs.  A work item
is (M-tile group, N tile); an iteration is (work item, voxel tile), items outer.  CTA c of P runs iterations
[c * T / P, (c + 1) * T / P): every iteration once, per-CTA work within one voxel tile, and in deterministic mode each CTA stores
into the slot of its rank among the CTAs of its item, below the route's split count."""
import math

import numpy as np
import pytest

import conv_route_cases as R
import plan_launches as P
import segresnet_cases as S


def pick_tile(w, h, d):
    """conv_common.cuh: pick_tile, the per-tap voxel tile of 128 output voxels"""
    tw = 8 if w >= 8 else 4 if w >= 4 else 2 if w >= 2 else 1
    rem = 128 // tw
    th = 4 if h >= 4 else 2 if h >= 2 else 1
    th = min(th, rem)
    return tw, th, rem // th


def kc_bucket(c):
    return 64 if c > 32 else 32 if c > 16 else 16


def bn_bucket(c):
    return 128 if c > 64 else kc_bucket(c)


CONFIGS = ("C2", "C3", "brats-dynunet", "brats-segresnet", "brats-segresnet-128")
CASES = sorted({(c, l.op, P.pad8(l.c), P.pad8(l.co), l.dims) for c in CONFIGS for l in P.BY_NAME[c].launches()
                if l.kernel == "wgrad"})


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


def sk_cta(x, T, P):
    """wgrad.cu: wgrad_sk_cta, the CTA that runs iteration x"""
    return ((x + 1) * P - 1) // T


def restate(op, ci, co, dims, num_sms, n=2):
    """the per-tap route fields wgrad_tiling computes, and the per-CTA ranges"""
    _, ksz, _ = R.wgrad_geometry(op, dims)
    d, h, w = dims
    tw, th, td = pick_tile(w, h, d)
    cb, bn = kc_bucket(ci), bn_bucket(co)
    units = ksz ** 3 * math.ceil(ci / cb)
    qtiles = math.ceil(units / (128 // cb))
    qt = min(2 * (128 // bn), qtiles)
    groups = math.ceil(qtiles / qt)
    qt = math.ceil(qtiles / groups)
    cotiles = math.ceil(co / bn)
    kblocks = n * math.ceil(d / td) * math.ceil(h / th) * math.ceil(w / tw)
    items = groups * cotiles
    T = items * kblocks
    P = min(num_sms, T)
    ranges = [(c * T // P, (c + 1) * T // P) for c in range(P)]
    first = [sk_cta(i * kblocks, T, P) for i in range(items)]
    last = [sk_cta((i + 1) * kblocks - 1, T, P) for i in range(items)]
    splits = max(l - f + 1 for f, l in zip(first, last))
    fields = dict(cb=cb, bn=bn, qt=qt, groups=groups, cotiles=cotiles, kblocks=kblocks, splits=splits, tw=tw, th=th, td=td,
                  ctas=P, part_bytes=splits * ksz ** 3 * ci * co * 4)
    return fields, ranges, first, T, kblocks


@pytest.mark.parametrize("num_sms", [114, 132])
@pytest.mark.parametrize("plan,op,ci,co,dims", CASES, ids=lambda v: str(v))
def test_streamk_partition(L, plan, op, ci, co, dims, num_sms):
    n = P.BY_NAME[plan].n
    for split in (False, True):
        r = R.wgrad_query(L, op, ci, co, dims, split, num_sms=num_sms, n=n)
        assert r is not None, (op, ci, co, dims)
        if r["kind"] != "tap":
            continue
        fields, ranges, first, T, kblocks = restate(op, ci, co, dims, num_sms, n=n)
        assert {k: r[k] for k in fields} == fields
        assert R.wgrad_query(L, op, ci, co, dims, split, deterministic=True, num_sms=num_sms, n=n) == r
        # every CTA of the machine works unless there are fewer iterations
        assert r["ctas"] == min(num_sms, T)
        # every (item, voxel tile) exactly once: the ranges tile [0, T) in order
        assert ranges[0][0] == 0 and ranges[-1][1] == T
        assert all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
        sizes = np.array([b - a for a, b in ranges])
        assert sizes.min() >= 1 and sizes.max() - sizes.min() <= 1
        assert all(sk_cta(a, T, len(ranges)) == c == sk_cta(b - 1, T, len(ranges)) for c, (a, b) in enumerate(ranges))
        # deterministic slots: the rank of each CTA among the CTAs of each item it touches is below splits, and the CTA that
        # runs an item's first iteration is rank 0
        for c, (a, b) in enumerate(ranges):
            for item in range(a // kblocks, (b - 1) // kblocks + 1):
                rank = c - first[item]
                assert 0 <= rank < r["splits"]
                assert sk_cta(item * kblocks, T, len(ranges)) == first[item]
                if a <= item * kblocks < b:
                    assert rank == 0


def test_wide_c2_launches_fill_every_sm(L):
    """the 3x3x3 launches of more than 64 input channels ran on 108 of 132 SMs before stream-K"""
    wide = [s[1:] for s in CASES if s[0] == "C2" and s[1] in ("k3s1", "k3s2") and s[2] > 64]
    assert len({s for s in wide}) >= 5
    for op, ci, co, dims in wide:
        r = R.wgrad_query(L, op, ci, co, dims)
        assert r["kind"] == "tap" and r["ctas"] == 132, (op, ci, co, dims, r)


@pytest.mark.parametrize("precision", ["bf16", "split"])
def test_segresnet_brats_wgrad_routes(L, precision):
    """the weight-gradient route of every SegResNet layer of the BraTS recipe on a 132-SM H100 (the table the at-size GPU test
    asserts), and the per-tap ones split over every SM"""
    assert S.wgrad_route_table(L, precision == "split") == S.BRATS_WGRAD_ROUTES[precision]
    for l in P.BY_NAME["brats-segresnet"].launches():
        if l.kernel == "wgrad":
            r = P.wgrad_route(L, l, precision == "split")
            assert r["ctas"] == 132, (l, r)
