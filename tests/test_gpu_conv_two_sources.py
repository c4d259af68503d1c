"""A fused 1x1x1 second source wider than the 3x3x3 first source (the last decoder level's conv2 with its `sample`): the K chunk
width follows the 3x3x3 source and the second source is walked in several chunks.  Checked against the fp64 oracle, and in bf16
bit for bit against the same convolution with the first source zero-padded to the second source's width, which sizes the
chunks to the wide source."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"
TOL_STORE = {False: 4e-3, True: 5e-5}      # rel-L2 of a stored activation: bf16 / hi+lo (as in test_gpu_ops.py)


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _pack(L, w, split):
    cout, cin, k = w.shape[0], w.shape[1], w.shape[2]
    hi, lo, cop, cip, _ = L.pack_weights(w, 0, split=split)
    q = hi.float() + (lo.float() if split else 0)
    return hi, lo, cop, cip, q.double().cpu()[:, :cout, :cin].reshape(k, k, k, cout, cin).permute(3, 4, 0, 1, 2)


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("ci", [16, 32])
@pytest.mark.parametrize("D", [8, 16])          # 8: per-tap tiles, 16: the halo kernel in bf16 (asserted below)
def test_wide_second_source_matches_oracle_and_padded_first_source(pkg, split, ci, D):
    L = pkg.lib
    torch.manual_seed(ci + D)
    n, ci2, co = 2, 64, 32
    h = torch.randn(n, ci, D, D, D, device=DEV)
    x = torch.randn(n, ci2, D, D, D, device=DEV)
    r = torch.randn(n, co, D, D, D, device=DEV)
    w2 = torch.randn(co, ci, 3, 3, 3, device=DEV) / (ci * 27) ** 0.5
    ws = torch.randn(co, ci2, 1, 1, 1, device=DEV) / ci2 ** 0.5
    ah, ax, res = (L.Act.from_ncdhw(t, split=split) for t in (h, x, r))
    w2h, w2l, cop, cip, w2q = _pack(L, w2, split)
    wsh, wsl, _, cips, wsq = _pack(L, ws, split)

    def run(a, wh, wl, cin_p, kind, kc):
        y = L.Act.empty(n, D, D, D, co, split=split)
        st = torch.zeros(n, co, 2, dtype=torch.float64, device=DEV)
        kw = dict(x2=ax, w2_hi=wsh, w2_lo=wsl, cip2=cips, res=res, stats=st, stats_ld=co)
        route = L.conv3d_route(a, wh, wl, 3, 1, y, cop, cin_p, **kw)
        assert (route["kind"], route["kc"], route["kchunks"]) == (kind, kc, (a.c // kc, ci2 // kc))
        L.conv3d(a, wh, wl, 3, 1, y, cop, cin_p, **kw)
        torch.cuda.synchronize()
        return y, st

    y, st = run(ah, w2h, w2l, cip, "halo" if D == 16 and not split else "tap", ci)
    ref = (F.conv3d(ah.to_ncdhw(ci).double().cpu(), w2q, padding=1) + F.conv3d(ax.to_ncdhw(ci2).double().cpu(), wsq)
           + res.to_ncdhw(co).double().cpu())
    assert rel(y.to_ncdhw(co), ref) < TOL_STORE[split]
    got = y.to_ncdhw(co).double().cpu()
    s_ref = torch.stack([got.sum(dim=(2, 3, 4)), (got * got).sum(dim=(2, 3, 4))], dim=-1)
    assert rel(st.cpu(), s_ref) < (2e-3 if not split else 1e-5)     # stats are taken before the bf16 rounding

    if split:
        return      # three passes per K chunk: the second source's passes interleave differently with narrower chunks
    zeros = torch.zeros(n, ci2 - ci, D, D, D, device=DEV)
    ahp = L.Act.from_ncdhw(torch.cat([ah.to_ncdhw(ci), zeros], dim=1))
    w2p = torch.cat([w2h.float()[:, :co, :ci].reshape(3, 3, 3, co, ci).permute(3, 4, 0, 1, 2),
                     torch.zeros(co, ci2 - ci, 3, 3, 3, device=DEV)], dim=1)
    w2ph, _, _, cipp, _ = L.pack_weights(w2p, 0)
    yp, stp = run(ahp, w2ph, None, cipp, "tap", 64)     # (KC = 64, BN = 32): per-tap tiles at any extent (halo_keeps_occupancy)
    assert int((y.hi != yp.hi).sum()) == 0
    # fp32 per-tile partial sums: at D = 16 the two launches tile the output differently
    assert float((st - stp).abs().max()) <= 1e-6 * float(stp.abs().max())
