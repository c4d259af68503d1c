"""The stream-K per-tap weight gradient (wgrad.cu: k_wgrad) against fp64, element by element with the bounds of
tests/test_gpu_conv_routes.py, in atomic and in deterministic mode: the wide 3x3x3 launches of the C2 step at their full
extents, a launch whose iterations do not divide evenly over the CTAs and whose work items span three or more CTAs, 1x1x1
launches whose work items have one M tile (the two consumer warpgroups split its voxel tiles), and split precision.
Deterministic results repeat bit for bit, computed into a partial buffer filled with NaN: the slots an item does not use must
be zeroed by the launch itself."""
import itertools

import pytest
import torch
import torch.nn.functional as F

import conv_route_cases as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
A_ACC = 2.0 ** -15                                # fp32 accumulation, relative to sum |a| |dy|

# (op, ci, co, dy extents, split)
WIDE_C2 = [("k3s1", 128, 128, (64, 64, 64), False), ("k3s1", 128, 128, (32, 32, 32), False),
           ("k3s1", 256, 256, (32, 32, 32), False), ("k3s1", 128, 256, (16, 16, 16), False),
           ("k3s1", 256, 256, (16, 16, 16), False), ("k3s2", 128, 128, (16, 16, 16), False)]
SINGLE_M_TILE = [("k1", 128, 32, (32, 32, 32), False), ("k1", 64, 128, (16, 16, 16), False), ("k1", 32, 64, (32, 32, 32), False),
                 ("k1", 24, 16, (9, 6, 5), False)]
SPLIT = [("k3s1", 128, 128, (16, 16, 16), True), ("k3s2", 256, 256, (8, 8, 8), True), ("k1", 128, 32, (16, 16, 16), True),
         ("k2s2", 64, 128, (8, 8, 8), True)]
CASES = WIDE_C2 + SINGLE_M_TILE + SPLIT


@pytest.fixture(scope="module")
def L(pkg):
    pkg.lib.load_library()
    return pkg.lib


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def stored(n, dims, c, split, gen):
    """random NDHWC activation -> (hi, lo or None, exact fp64 value)"""
    v = torch.randn(n, *dims, c, generator=gen, device=DEV)
    hi = v.bfloat16()
    lo = (v - hi.float()).bfloat16() if split else None
    return hi, lo, hi.double() + (lo.double() if split else 0)


def wgrad64(a, dy, ksz, stride, pad):
    """dw[kd * k^2 + kh * k + kw][ci][co] = sum over n and the output voxels v of a[v * stride + tap - pad][ci] dy[v][co], NDHWC"""
    n, d, h, w, co = dy.shape
    ap = F.pad(a, (0, 0) + (pad, pad) * 3)
    out = []
    for kd, kh, kw in itertools.product(range(ksz), repeat=3):
        sl = ap[:, kd:kd + stride * (d - 1) + 1:stride, kh:kh + stride * (h - 1) + 1:stride, kw:kw + stride * (w - 1) + 1:stride]
        out.append(sl.reshape(-1, a.shape[-1]).T @ dy.reshape(-1, co))
    return torch.stack(out)


def check(got, ref, bound, what):
    err = (got.double() - ref).abs()
    lim = 2.0 ** -20 * ref.abs() + bound + 1e-30
    bad = err > lim
    if bool(bad.any()):
        idx = tuple(int(i) for i in bad.nonzero()[0])
        pytest.fail("%s: %d of %d elements out of bounds; first at %s (tap, ci, co): got %.8g ref %.8g bound %.3g"
                    % (what, int(bad.sum()), bad.numel(), idx, float(got[idx]), float(ref[idx]), float(lim[idx])))


@pytest.mark.parametrize("op,ci,co,dims,split", CASES, ids=lambda v: str(v))
def test_streamk_wgrad_matches_fp64(L, op, ci, co, dims, split):
    n = 2
    adims, ksz, stride = R.wgrad_geometry(op, dims)
    pad = 0 if ksz == 2 else ksz // 2
    gen = torch.Generator(device=DEV).manual_seed(ci * 1000 + co + sum(dims))
    ahi, alo, av = stored(n, adims, ci, split, gen)
    yhi, ylo, yv = stored(n, dims, co, split, gen)
    a, dy = L.Act(ahi, alo), L.Act(yhi, ylo)
    ref = wgrad64(av, yv, ksz, stride, pad)
    bound = A_ACC * wgrad64(av.abs(), yv.abs(), ksz, stride, pad)
    del av, yv
    T = ksz ** 3

    r = L.wgrad_route(a, dy, ksz, stride, ci, co, num_sms=sms())
    assert r["kind"] == "tap" and r["npass"] == (3 if split else 1), r
    iters = r["groups"] * r["cotiles"] * r["kblocks"]
    assert r["ctas"] == min(sms(), iters), r
    if (op, ci, co, dims) == ("k3s1", 128, 128, (16, 16, 16)):   # uneven ranges, and work items over three or more CTAs
        assert iters % r["ctas"] != 0 and r["splits"] >= 3, r
    if op == "k1":
        assert r["groups"] == 1 and r["qt"] == 1, r

    dw = torch.zeros(T, ci, co, device=DEV)
    assert L.wgrad_ex(a, dy, ksz, stride, ci, co, dw) == 0
    torch.cuda.synchronize()
    check(dw, ref, bound, "dw (atomics)")

    rd = L.wgrad_route(a, dy, ksz, stride, ci, co, deterministic=True, num_sms=sms())
    assert rd == r
    outs = []
    for _ in range(2):
        part = torch.full((rd["part_bytes"] // 4,), float("nan"), device=DEV)
        dwd = torch.full((T, ci, co), float("nan"), device=DEV)
        assert L.wgrad_ex(a, dy, ksz, stride, ci, co, dwd, part=part) == rd["splits"]
        torch.cuda.synchronize()
        outs.append(dwd)
    assert torch.equal(outs[0], outs[1]), "deterministic weight gradient differs between two runs"
    check(outs[0], ref, bound, "dw (deterministic)")
