"""Kernel routes of the convolution and the weight gradient, and one test case per route.

A route is the kernel a launch runs on: kind (per-tap tiles, halo box, parity class 1 or 2) with its N tile BN and K chunk KC
for the convolution, or kind (SIMT, per-tap, halo) with its CB / BN for the weight gradient, in each precision, epilogue mode
and number of sources.  The library reports the route it takes (include/b200unet_diag.h); the host tests sweep that query over
the shapes the plans can launch and require every reachable route to have a case below, and the GPU tests run every case
against an fp64 reference after checking that it still takes its route.  The query reads shapes and which pointers are NULL,
so the sweep passes placeholder addresses.
"""
import itertools
from dataclasses import dataclass
from typing import Tuple

CHANNELS = (8, 16, 24, 32, 40, 64, 72, 128, 192, 256)
SMALL_PLANE = (3, 5, 7)        # output extents (d, h, w): per-tap tiles only
LARGE_PLANE = (2, 16, 8)       # output plane of at least 8 x 16: fills the halo tile


def kc_of(c: int) -> int:
    """K chunk of a source with c channels"""
    return 64 if c > 32 else 32 if c > 16 else 16


# --------------------------------------------------------------------------------------------- placeholders for host queries
class ShapeAct:
    """an activation view with the shape of lib.Act and placeholder (never dereferenced) addresses"""

    def __init__(self, L, n, d, h, w, c, split=False):
        self.L, self.n, self.d, self.h, self.w, self.c, self.ld, self.split = L, n, d, h, w, c, c, split

    def ct(self):
        t = self.L.Tensor5()
        t.hi = 0x10000
        t.lo = 0x20000 if self.split else None
        t.n, t.d, t.h, t.w, t.c, t.ld = self.n, self.d, self.h, self.w, self.c, self.ld
        return t


class Addr:
    """stands in for a device tensor whose address is all the query looks at"""

    def data_ptr(self):
        return 0x30000


# ---------------------------------------------------------------------------------------------------------- convolution
@dataclass(frozen=True)
class ConvCase:
    """op: k3s1 | k3s2 | k1 (forward conv), class1 (data gradient of a k3s2 conv: source = dY at half the output extent) or
    class2 (ConvTranspose3d, kernel = stride = 2).  cin / cout: channels of source 0 / of the output view; cin2 > 0 adds a
    fused 1x1x1 second source; dims: output extents (d, h, w).  The remaining fields are the route it must take."""
    kind: str
    bn: int
    kc: int
    split: bool
    mode: int
    nsrc: int
    op: str
    cin: int
    cout: int
    dims: Tuple[int, int, int]
    cin2: int = 0
    kchunks: Tuple[int, int] = (1, 0)

    @property
    def key(self):
        return conv_key(self.kind, self.bn, self.kc, self.split, self.mode, self.nsrc)

    @property
    def id(self):
        return "%s-bn%d-kc%d-%s-m%d-s%d" % (self.kind, self.bn, self.kc, "split" if self.split else "bf16", self.mode, self.nsrc)


def conv_key(kind, bn, kc, split, mode, nsrc):
    return (kind, bn, kc, "split" if split else "bf16", mode, nsrc)


def conv_geometry(op, cin, dims):
    """(source extents, ksz, stride, cls_mode) of a case's source 0 for output extents dims"""
    d, h, w = dims
    if op == "k3s1":
        return (d, h, w), 3, 1, 0
    if op == "k1":
        return (d, h, w), 1, 1, 0
    if op == "k3s2":
        return (2 * d, 2 * h, 2 * w), 3, 2, 0
    if op == "class1":
        return (d // 2, h // 2, w // 2), 3, 1, 1
    if op == "class2":
        return (d // 2, h // 2, w // 2), 2, 2, 2
    if op == "k2s2":   # unpadded kernel = stride 2 (the data gradient of a kernel-2 transposed convolution)
        return (2 * d, 2 * h, 2 * w), 2, 2, 0
    raise ValueError(op)


def conv_query(L, op, cin, cout, dims, split=False, mode=0, cin2=0, n=2, lo_out=False):
    """route of a convolution of this shape (host-only); None when the library refuses the combination.  The output has a lo
    plane in split precision, and with lo_out also for bf16 operands (the fp32 accumulators stored as hi + lo)."""
    sdims, ksz, stride, cls = conv_geometry(op, cin, dims)
    x = ShapeAct(L, n, *sdims, cin, split)
    out = ShapeAct(L, n, *dims, cout, split or lo_out)
    w = Addr()
    wl = Addr() if split else None
    kw = dict(cls_mode=cls, mode=mode)
    if cin2:
        kw.update(x2=ShapeAct(L, n, *dims, cin2, split), w2_hi=w, w2_lo=wl, cip2=cin2)
    if mode == 1:
        kw.update(gn_x=ShapeAct(L, n, *dims, cout, split), coef=Addr(), coef_ld=cout, bstats=Addr())
    try:
        return L.conv3d_route(x, w, wl, ksz, stride, out, cout, cin, **kw)
    except RuntimeError:
        return None


def conv_sweep(L):
    """every (shape, options, route) of the sweep: yields (params dict, route dict)"""
    ops = {"k3s1": (SMALL_PLANE, LARGE_PLANE), "k3s2": (SMALL_PLANE, LARGE_PLANE), "k1": (SMALL_PLANE, LARGE_PLANE),
           "class1": ((4, 6, 8), (2, 32, 16)), "class2": ((4, 6, 8), (2, 32, 16))}
    for op, planes in ops.items():
        second = (0,) if op.startswith("class") else (0,) + CHANNELS
        for dims, cin, cout, cin2, split, mode in itertools.product(planes, CHANNELS, CHANNELS, second, (False, True), (0, 1)):
            r = conv_query(L, op, cin, cout, dims, split, mode, cin2)
            if r is not None:
                yield dict(op=op, dims=dims, cin=cin, cout=cout, cin2=cin2, split=split, mode=mode), r


def route_key_of(params, r):
    return conv_key(r["kind"], r["bn"], r["kc"], params["split"], params["mode"], 2 if params["cin2"] else 1)


# Shapes: output extents not multiples of the tile (per-tap 8 x 4 x 4 and halo 8 x 16 x 1 tiles; class tiles on the half-size
# grid), batch 2, and a partial last N tile where the bucket allows it (cout 8 of BN 16, 24 of 32, 40 or 72 of 64, 200 of 128).
P = (5, 6, 9)          # per-tap plane
H = (3, 18, 10)        # halo plane
S2 = (3, 5, 7)         # stride-2 output (source 6 x 10 x 14)
CL = (6, 10, 18)       # class-mode output (source 3 x 5 x 9)
_C = ConvCase
CONV_CASES = [
    _C("tap", 16, 16, False, 0, 1, "k3s2", 16, 8, S2),
    _C("tap", 16, 16, False, 0, 2, "k3s1", 16, 8, P, cin2=64, kchunks=(1, 4)),
    _C("tap", 16, 16, False, 1, 1, "k3s1", 8, 8, P),
    _C("tap", 16, 16, False, 1, 2, "k3s2", 16, 8, S2, cin2=8, kchunks=(1, 1)),
    _C("tap", 16, 16, True, 0, 1, "k1", 16, 8, P),
    _C("tap", 16, 16, True, 0, 2, "k3s1", 8, 8, P, cin2=64, kchunks=(1, 4)),
    _C("tap", 16, 16, True, 1, 1, "k3s2", 16, 8, S2),
    _C("tap", 16, 16, True, 1, 2, "k3s1", 16, 8, P, cin2=8, kchunks=(1, 1)),
    _C("tap", 16, 32, False, 0, 1, "k3s1", 24, 8, P),
    _C("tap", 16, 32, False, 0, 2, "k3s2", 24, 8, S2, cin2=40, kchunks=(1, 2)),
    _C("tap", 16, 32, False, 1, 1, "k1", 24, 8, P),
    _C("tap", 16, 32, False, 1, 2, "k3s1", 24, 8, P, cin2=16, kchunks=(1, 1)),
    _C("tap", 16, 32, True, 0, 1, "k3s2", 24, 8, S2),
    _C("tap", 16, 32, True, 0, 2, "k3s1", 24, 8, P, cin2=40, kchunks=(1, 2)),
    _C("tap", 16, 32, True, 1, 1, "k3s1", 24, 8, P),
    _C("tap", 16, 32, True, 1, 2, "k3s2", 24, 8, S2, cin2=16, kchunks=(1, 1)),
    _C("tap", 16, 64, False, 0, 1, "k1", 136, 8, P, kchunks=(3, 0)),
    _C("tap", 16, 64, False, 0, 2, "k3s1", 40, 8, P, cin2=72, kchunks=(1, 2)),
    _C("tap", 16, 64, False, 1, 1, "k3s2", 72, 8, S2, kchunks=(2, 0)),
    _C("tap", 16, 64, False, 1, 2, "k3s1", 40, 8, P, cin2=24, kchunks=(1, 1)),
    _C("tap", 16, 64, True, 0, 1, "k3s1", 40, 8, P),
    _C("tap", 16, 64, True, 0, 2, "k3s2", 40, 8, S2, cin2=72, kchunks=(1, 2)),
    _C("tap", 16, 64, True, 1, 1, "k1", 72, 8, P, kchunks=(2, 0)),
    _C("tap", 16, 64, True, 1, 2, "k3s1", 40, 8, P, cin2=24, kchunks=(1, 1)),
    _C("tap", 32, 16, False, 0, 1, "k3s2", 16, 24, S2),
    _C("tap", 32, 16, False, 0, 2, "k3s1", 16, 24, P, cin2=64, kchunks=(1, 4)),
    _C("tap", 32, 16, False, 1, 1, "k3s1", 8, 24, P),
    _C("tap", 32, 16, False, 1, 2, "k3s2", 16, 24, S2, cin2=8, kchunks=(1, 1)),
    _C("tap", 32, 16, True, 0, 1, "k1", 16, 24, P),
    _C("tap", 32, 16, True, 0, 2, "k3s1", 8, 24, P, cin2=64, kchunks=(1, 4)),
    _C("tap", 32, 16, True, 1, 1, "k3s2", 16, 24, S2),
    _C("tap", 32, 16, True, 1, 2, "k3s1", 16, 24, P, cin2=8, kchunks=(1, 1)),
    _C("tap", 32, 32, False, 0, 1, "k3s1", 24, 24, P),
    _C("tap", 32, 32, False, 0, 2, "k3s2", 24, 24, S2, cin2=40, kchunks=(1, 2)),
    _C("tap", 32, 32, False, 1, 1, "k1", 24, 24, P),
    _C("tap", 32, 32, False, 1, 2, "k3s1", 24, 24, P, cin2=16, kchunks=(1, 1)),
    _C("tap", 32, 32, True, 0, 1, "k3s2", 24, 24, S2),
    _C("tap", 32, 32, True, 0, 2, "k3s1", 24, 24, P, cin2=40, kchunks=(1, 2)),
    _C("tap", 32, 32, True, 1, 1, "k3s1", 24, 24, P),
    _C("tap", 32, 32, True, 1, 2, "k3s2", 24, 24, S2, cin2=16, kchunks=(1, 1)),
    _C("tap", 32, 64, False, 0, 1, "k1", 136, 24, P, kchunks=(3, 0)),
    _C("tap", 32, 64, False, 0, 2, "k3s1", 40, 24, P, cin2=72, kchunks=(1, 2)),
    _C("tap", 32, 64, False, 1, 1, "k3s2", 72, 24, S2, kchunks=(2, 0)),
    _C("tap", 32, 64, False, 1, 2, "k3s1", 40, 24, P, cin2=24, kchunks=(1, 1)),
    _C("tap", 32, 64, True, 0, 1, "k3s1", 40, 24, P),
    _C("tap", 32, 64, True, 0, 2, "k3s2", 40, 24, S2, cin2=72, kchunks=(1, 2)),
    _C("tap", 32, 64, True, 1, 1, "k1", 72, 24, P, kchunks=(2, 0)),
    _C("tap", 32, 64, True, 1, 2, "k3s1", 40, 24, P, cin2=24, kchunks=(1, 1)),
    _C("tap", 64, 16, False, 0, 1, "k3s2", 16, 40, S2),
    _C("tap", 64, 16, False, 0, 2, "k3s1", 16, 40, P, cin2=64, kchunks=(1, 4)),
    _C("tap", 64, 16, False, 1, 1, "k3s1", 8, 40, P),
    _C("tap", 64, 16, False, 1, 2, "k3s2", 16, 40, S2, cin2=8, kchunks=(1, 1)),
    _C("tap", 64, 16, True, 0, 1, "k1", 16, 40, P),
    _C("tap", 64, 16, True, 0, 2, "k3s1", 8, 40, P, cin2=64, kchunks=(1, 4)),
    _C("tap", 64, 16, True, 1, 1, "k3s2", 16, 40, S2),
    _C("tap", 64, 16, True, 1, 2, "k3s1", 16, 40, P, cin2=8, kchunks=(1, 1)),
    _C("tap", 64, 32, False, 0, 1, "k3s1", 24, 40, P),
    _C("tap", 64, 32, False, 0, 2, "k3s2", 24, 40, S2, cin2=40, kchunks=(1, 2)),
    _C("tap", 64, 32, False, 1, 1, "k1", 24, 40, P),
    _C("tap", 64, 32, False, 1, 2, "k3s1", 24, 40, P, cin2=16, kchunks=(1, 1)),
    _C("tap", 64, 32, True, 0, 1, "k3s2", 24, 40, S2),
    _C("tap", 64, 32, True, 0, 2, "k3s1", 24, 40, P, cin2=40, kchunks=(1, 2)),
    _C("tap", 64, 32, True, 1, 1, "k3s1", 24, 40, P),
    _C("tap", 64, 32, True, 1, 2, "k3s2", 24, 40, S2, cin2=16, kchunks=(1, 1)),
    _C("tap", 64, 64, False, 0, 1, "k1", 136, 40, P, kchunks=(3, 0)),
    _C("tap", 64, 64, False, 0, 2, "k3s1", 40, 40, P, cin2=72, kchunks=(1, 2)),
    _C("tap", 64, 64, False, 1, 1, "k3s2", 72, 40, S2, kchunks=(2, 0)),
    _C("tap", 64, 64, False, 1, 2, "k3s1", 40, 40, P, cin2=24, kchunks=(1, 1)),
    _C("tap", 64, 64, True, 0, 1, "k3s1", 40, 40, P),
    _C("tap", 64, 64, True, 0, 2, "k3s2", 40, 40, S2, cin2=72, kchunks=(1, 2)),
    _C("tap", 64, 64, True, 1, 1, "k1", 72, 40, P, kchunks=(2, 0)),
    _C("tap", 64, 64, True, 1, 2, "k3s1", 40, 40, P, cin2=24, kchunks=(1, 1)),
    _C("tap", 128, 16, False, 0, 1, "k3s2", 16, 200, S2),
    _C("tap", 128, 16, False, 0, 2, "k3s1", 16, 200, P, cin2=64, kchunks=(1, 4)),
    _C("tap", 128, 16, False, 1, 1, "k3s1", 8, 200, P),
    _C("tap", 128, 16, False, 1, 2, "k3s2", 16, 200, S2, cin2=8, kchunks=(1, 1)),
    _C("tap", 128, 16, True, 0, 1, "k1", 16, 200, P),
    _C("tap", 128, 16, True, 0, 2, "k3s1", 8, 200, P, cin2=64, kchunks=(1, 4)),
    _C("tap", 128, 16, True, 1, 1, "k3s2", 16, 200, S2),
    _C("tap", 128, 16, True, 1, 2, "k3s1", 16, 200, P, cin2=8, kchunks=(1, 1)),
    _C("tap", 128, 32, False, 0, 1, "k3s1", 24, 200, P),
    _C("tap", 128, 32, False, 0, 2, "k3s2", 24, 200, S2, cin2=40, kchunks=(1, 2)),
    _C("tap", 128, 32, False, 1, 1, "k1", 24, 200, P),
    _C("tap", 128, 32, False, 1, 2, "k3s1", 24, 200, P, cin2=16, kchunks=(1, 1)),
    _C("tap", 128, 32, True, 0, 1, "k3s2", 24, 200, S2),
    _C("tap", 128, 32, True, 0, 2, "k3s1", 24, 200, P, cin2=40, kchunks=(1, 2)),
    _C("tap", 128, 32, True, 1, 1, "k3s1", 24, 200, P),
    _C("tap", 128, 32, True, 1, 2, "k3s2", 24, 200, S2, cin2=16, kchunks=(1, 1)),
    _C("tap", 128, 64, False, 0, 1, "k1", 136, 200, P, kchunks=(3, 0)),
    _C("tap", 128, 64, False, 0, 2, "k3s1", 40, 200, P, cin2=72, kchunks=(1, 2)),
    _C("tap", 128, 64, False, 1, 1, "k3s2", 72, 200, S2, kchunks=(2, 0)),
    _C("tap", 128, 64, False, 1, 2, "k3s1", 40, 200, P, cin2=24, kchunks=(1, 1)),
    _C("tap", 128, 64, True, 0, 1, "k3s1", 40, 200, P),
    _C("tap", 128, 64, True, 0, 2, "k3s2", 40, 200, S2, cin2=72, kchunks=(1, 2)),
    _C("tap", 128, 64, True, 1, 1, "k1", 72, 200, P, kchunks=(2, 0)),
    _C("tap", 128, 64, True, 1, 2, "k3s1", 40, 200, P, cin2=24, kchunks=(1, 1)),
    _C("halo", 16, 16, False, 0, 1, "k3s1", 16, 8, H),
    _C("halo", 16, 16, False, 0, 2, "k3s1", 16, 8, H, cin2=64, kchunks=(1, 4)),
    _C("halo", 16, 16, False, 1, 1, "k3s1", 8, 8, H),
    _C("halo", 16, 16, False, 1, 2, "k3s1", 16, 8, H, cin2=8, kchunks=(1, 1)),
    _C("halo", 16, 32, False, 0, 1, "k3s1", 24, 8, H),
    _C("halo", 16, 32, False, 0, 2, "k3s1", 24, 8, H, cin2=40, kchunks=(1, 2)),
    _C("halo", 16, 32, False, 1, 1, "k3s1", 24, 8, H),
    _C("halo", 16, 32, False, 1, 2, "k3s1", 24, 8, H, cin2=16, kchunks=(1, 1)),
    _C("halo", 32, 16, False, 0, 1, "k3s1", 8, 24, H),
    _C("halo", 32, 16, False, 0, 2, "k3s1", 16, 24, H, cin2=64, kchunks=(1, 4)),
    _C("halo", 32, 16, False, 1, 1, "k3s1", 16, 24, H),
    _C("halo", 32, 16, False, 1, 2, "k3s1", 8, 24, H, cin2=8, kchunks=(1, 1)),
    _C("halo", 32, 32, False, 0, 1, "k3s1", 24, 24, H),
    _C("halo", 32, 32, False, 0, 2, "k3s1", 24, 24, H, cin2=40, kchunks=(1, 2)),
    _C("halo", 32, 32, False, 1, 1, "k3s1", 24, 24, H),
    _C("halo", 32, 32, False, 1, 2, "k3s1", 24, 24, H, cin2=16, kchunks=(1, 1)),
    _C("halo", 64, 16, False, 0, 1, "k3s1", 16, 40, H),
    _C("halo", 64, 16, False, 0, 2, "k3s1", 8, 40, H, cin2=64, kchunks=(1, 4)),
    _C("halo", 64, 16, False, 1, 1, "k3s1", 16, 40, H),
    _C("halo", 64, 16, False, 1, 2, "k3s1", 16, 40, H, cin2=8, kchunks=(1, 1)),
    _C("halo", 64, 32, False, 0, 1, "k3s1", 24, 40, H),
    _C("halo", 64, 32, False, 0, 2, "k3s1", 24, 40, H, cin2=40, kchunks=(1, 2)),
    _C("halo", 64, 32, False, 1, 1, "k3s1", 24, 40, H),
    _C("halo", 64, 32, False, 1, 2, "k3s1", 24, 40, H, cin2=16, kchunks=(1, 1)),
    _C("halo", 64, 64, False, 0, 1, "k3s1", 64, 40, H),
    _C("halo", 64, 64, False, 0, 2, "k3s1", 40, 40, H, cin2=72, kchunks=(1, 2)),
    _C("halo", 64, 64, False, 1, 1, "k3s1", 40, 40, H),
    _C("halo", 64, 64, False, 1, 2, "k3s1", 40, 40, H, cin2=24, kchunks=(1, 1)),
    _C("halo", 128, 16, False, 0, 1, "k3s1", 16, 200, H),
    _C("halo", 128, 16, False, 0, 2, "k3s1", 8, 200, H, cin2=64, kchunks=(1, 4)),
    _C("halo", 128, 16, False, 1, 1, "k3s1", 16, 200, H),
    _C("halo", 128, 16, False, 1, 2, "k3s1", 16, 200, H, cin2=8, kchunks=(1, 1)),
    _C("halo", 128, 32, False, 0, 1, "k3s1", 24, 200, H),
    _C("halo", 128, 32, False, 0, 2, "k3s1", 24, 200, H, cin2=40, kchunks=(1, 2)),
    _C("halo", 128, 32, False, 1, 1, "k3s1", 24, 200, H),
    _C("halo", 128, 32, False, 1, 2, "k3s1", 24, 200, H, cin2=16, kchunks=(1, 1)),
    _C("halo", 128, 64, False, 0, 1, "k3s1", 64, 200, H),
    _C("halo", 128, 64, False, 0, 2, "k3s1", 40, 200, H, cin2=72, kchunks=(1, 2)),
    _C("halo", 128, 64, False, 1, 1, "k3s1", 40, 200, H),
    _C("halo", 128, 64, False, 1, 2, "k3s1", 40, 200, H, cin2=24, kchunks=(1, 1)),
    _C("class1", 16, 16, False, 0, 1, "class1", 16, 8, CL),
    _C("class1", 16, 16, True, 0, 1, "class1", 8, 8, CL),
    _C("class1", 16, 32, False, 0, 1, "class1", 24, 8, CL),
    _C("class1", 16, 32, True, 0, 1, "class1", 24, 8, CL),
    _C("class1", 16, 64, False, 0, 1, "class1", 72, 8, CL, kchunks=(2, 0)),
    _C("class1", 16, 64, True, 0, 1, "class1", 40, 8, CL),
    _C("class1", 32, 16, False, 0, 1, "class1", 16, 24, CL),
    _C("class1", 32, 16, True, 0, 1, "class1", 8, 24, CL),
    _C("class1", 32, 32, False, 0, 1, "class1", 24, 24, CL),
    _C("class1", 32, 32, True, 0, 1, "class1", 24, 24, CL),
    _C("class1", 32, 64, False, 0, 1, "class1", 72, 24, CL, kchunks=(2, 0)),
    _C("class1", 32, 64, True, 0, 1, "class1", 40, 24, CL),
    _C("class1", 64, 16, False, 0, 1, "class1", 16, 72, CL),
    _C("class1", 64, 16, True, 0, 1, "class1", 8, 40, CL),
    _C("class1", 64, 32, False, 0, 1, "class1", 24, 72, CL),
    _C("class1", 64, 32, True, 0, 1, "class1", 24, 40, CL),
    _C("class1", 64, 64, False, 0, 1, "class1", 72, 72, CL, kchunks=(2, 0)),
    _C("class1", 64, 64, True, 0, 1, "class1", 40, 40, CL),
    _C("class2", 16, 16, False, 0, 1, "class2", 16, 8, CL),
    _C("class2", 16, 16, True, 0, 1, "class2", 8, 8, CL),
    _C("class2", 16, 32, False, 0, 1, "class2", 24, 8, CL),
    _C("class2", 16, 32, True, 0, 1, "class2", 24, 8, CL),
    _C("class2", 16, 64, False, 0, 1, "class2", 72, 8, CL, kchunks=(2, 0)),
    _C("class2", 16, 64, True, 0, 1, "class2", 40, 8, CL),
    _C("class2", 32, 16, False, 0, 1, "class2", 16, 24, CL),
    _C("class2", 32, 16, True, 0, 1, "class2", 8, 24, CL),
    _C("class2", 32, 32, False, 0, 1, "class2", 24, 24, CL),
    _C("class2", 32, 32, True, 0, 1, "class2", 24, 24, CL),
    _C("class2", 32, 64, False, 0, 1, "class2", 72, 24, CL, kchunks=(2, 0)),
    _C("class2", 32, 64, True, 0, 1, "class2", 40, 24, CL),
    _C("class2", 64, 16, False, 0, 1, "class2", 16, 72, CL),
    _C("class2", 64, 16, True, 0, 1, "class2", 8, 40, CL),
    _C("class2", 64, 32, False, 0, 1, "class2", 24, 72, CL),
    _C("class2", 64, 32, True, 0, 1, "class2", 24, 40, CL),
    _C("class2", 64, 64, False, 0, 1, "class2", 72, 72, CL, kchunks=(2, 0)),
    _C("class2", 64, 64, True, 0, 1, "class2", 40, 40, CL),
]

# Deep K loops: the route key leaves out how many K chunks a launch walks, and the cases above walk at most four (256 channels
# of KC 16, 136 of KC 64).  The C5 network's 384- and 768-channel layers walk 6 and 12 chunks of 64 channels, the BraTS DynUNet's
# up to 6; these cases walk 6, 7, 12 and 13 (392 and 776 channels: a partial last chunk), in both precisions and both epilogues,
# on the second source too, and through the parity-class kernels.  test_conv_routes_host.py requires a case here or above that
# walks at least as many chunks as any layer of the configurations the repository restates.
DEEP_K_CASES = [
    _C("tap", 64, 64, False, 0, 1, "k3s1", 776, 40, P, kchunks=(13, 0)),
    _C("tap", 128, 64, False, 0, 1, "k3s1", 384, 200, P, kchunks=(6, 0)),
    _C("tap", 64, 64, False, 0, 2, "k3s1", 384, 40, P, cin2=776, kchunks=(6, 13)),
    _C("tap", 64, 64, True, 0, 1, "k3s1", 768, 40, P, kchunks=(12, 0)),
    _C("tap", 64, 64, True, 0, 2, "k3s1", 392, 40, P, cin2=392, kchunks=(7, 7)),
    _C("tap", 64, 64, False, 1, 1, "k3s1", 768, 40, P, kchunks=(12, 0)),
    _C("tap", 64, 64, True, 1, 1, "k3s1", 392, 40, P, kchunks=(7, 0)),
    _C("class1", 64, 64, False, 0, 1, "class1", 392, 72, CL, kchunks=(7, 0)),
    _C("class1", 64, 64, True, 0, 1, "class1", 392, 40, CL, kchunks=(7, 0)),
    _C("class2", 64, 64, False, 0, 1, "class2", 392, 72, CL, kchunks=(7, 0)),
    _C("class2", 64, 64, True, 0, 1, "class2", 392, 40, CL, kchunks=(7, 0)),
]


def deep_k_id(case):
    return "%s-cin%d%s" % (case.id, case.cin, "+%d" % case.cin2 if case.cin2 else "")


# (kind, BN, KC) combinations B200_CONV_CONFIGS instantiates for no reachable launch, and why
CONV_UNREACHABLE = {
    ("halo", 16, 64): "the halo box would cost this configuration the second CTA per SM that per-tap tiles give it (halo_keeps_occupancy)",
    ("halo", 32, 64): "the halo box would cost this configuration the second CTA per SM that per-tap tiles give it (halo_keeps_occupancy)",
    ("class1", 128, 16): "class mode clamps BN to 64: its output staging tile sits beside the accumulator tile",
    ("class1", 128, 32): "class mode clamps BN to 64: its output staging tile sits beside the accumulator tile",
    ("class1", 128, 64): "class mode clamps BN to 64: its output staging tile sits beside the accumulator tile",
    ("class2", 128, 16): "class mode clamps BN to 64: its output staging tile sits beside the accumulator tile",
    ("class2", 128, 32): "class mode clamps BN to 64: its output staging tile sits beside the accumulator tile",
    ("class2", 128, 64): "class mode clamps BN to 64: its output staging tile sits beside the accumulator tile",
}


# ------------------------------------------------------------------------------------------------------ weight gradient
@dataclass(frozen=True)
class WgradCase:
    """op: k3s1 | k3s2 | k1 | k2s2 (the kernel = stride ConvTranspose3d); ci / co: channels of the activation / of dy;
    dims: extents of dy.  The remaining fields are the route of the atomic launch (the deterministic launch of a SIMT case runs
    on per-tap tiles, CB 16)."""
    kind: str
    cb: int             # SIMT: input channels / 8
    bn: int             # SIMT: 0
    split: bool
    op: str
    ci: int
    co: int
    dims: Tuple[int, int, int]

    @property
    def key(self):
        return wgrad_key(self.kind, self.cb, self.bn, self.split)

    @property
    def id(self):
        return "%s-cb%d-bn%d-%s" % (self.kind, self.cb, self.bn, "split" if self.split else "bf16")


def wgrad_key(kind, cb, bn, split):
    return (kind, cb, bn, "split" if split else "bf16")


def wgrad_geometry(op, dims):
    """(activation extents, ksz, stride) for dy extents dims"""
    d, h, w = dims
    if op in ("k3s1", "k1"):
        return dims, (3 if op == "k3s1" else 1), 1
    if op in ("k3s2", "k2s2"):
        return (2 * d, 2 * h, 2 * w), (3 if op == "k3s2" else 2), 2
    raise ValueError(op)


def wgrad_query(L, op, ci, co, dims, split=False, deterministic=False, num_sms=132, n=2):
    adims, ksz, stride = wgrad_geometry(op, dims)
    a = ShapeAct(L, n, *adims, ci, split)
    dy = ShapeAct(L, n, *dims, co, split)
    try:
        return L.wgrad_route(a, dy, ksz, stride, ci, co, deterministic=deterministic, num_sms=num_sms)
    except RuntimeError:
        return None


def wgrad_route_key(split, r):
    if r["kind"] == "simt":
        return wgrad_key("simt", r["ci8"], 0, split)
    return wgrad_key(r["kind"], r["cb"], r["bn"], split)


def wgrad_sweep(L, num_sms=132):
    for op, dims, ci, co, split, det in itertools.product(("k3s1", "k3s2", "k1", "k2s2"), (SMALL_PLANE, LARGE_PLANE), CHANNELS,
                                                          CHANNELS, (False, True), (False, True)):
        r = wgrad_query(L, op, ci, co, dims, split, det, num_sms)
        if r is not None:
            yield dict(op=op, dims=dims, ci=ci, co=co, split=split, deterministic=det), r


WP = (5, 6, 9)          # per-tap voxel tiles 8 x 4 x 4, partial on every axis
WH = (3, 18, 10)        # halo tiles 8 x 16 x 1, partial in h and w
_W = WgradCase
WGRAD_CASES = [
    _W("simt", 1, 0, False, "k1", 8, 32, WP),
    _W("simt", 1, 0, True, "k1", 8, 32, WP),
    _W("simt", 2, 0, False, "k1", 16, 64, WP),
    _W("simt", 2, 0, True, "k1", 16, 64, WP),
    _W("tap", 16, 16, False, "k3s2", 16, 8, WP),
    _W("tap", 16, 16, True, "k2s2", 8, 8, WP),
    _W("tap", 16, 32, False, "k3s1", 16, 24, WP),
    _W("tap", 16, 32, True, "k3s1", 16, 24, WP),
    _W("tap", 16, 64, False, "k3s2", 8, 40, WP),
    _W("tap", 16, 64, True, "k2s2", 16, 40, WP),
    _W("tap", 16, 128, False, "k3s1", 16, 200, WP),
    _W("tap", 16, 128, True, "k3s1", 8, 200, WP),
    _W("tap", 32, 16, False, "k3s2", 24, 8, WP),
    _W("tap", 32, 16, True, "k2s2", 24, 8, WP),
    _W("tap", 32, 32, False, "k3s1", 24, 24, WP),
    _W("tap", 32, 32, True, "k3s1", 24, 24, WP),
    _W("tap", 32, 64, False, "k3s2", 24, 40, WP),
    _W("tap", 32, 64, True, "k2s2", 24, 40, WP),
    _W("tap", 32, 128, False, "k3s1", 24, 200, WP),
    _W("tap", 32, 128, True, "k3s1", 24, 200, WP),
    _W("tap", 64, 16, False, "k3s2", 136, 8, WP),
    _W("tap", 64, 16, True, "k2s2", 40, 8, WP),
    _W("tap", 64, 32, False, "k3s1", 136, 24, WP),
    _W("tap", 64, 32, True, "k3s1", 40, 24, WP),
    _W("tap", 64, 64, False, "k3s2", 136, 40, WP),
    _W("tap", 64, 64, True, "k2s2", 40, 40, WP),
    _W("tap", 64, 128, False, "k3s1", 136, 200, WP),
    _W("tap", 64, 128, True, "k3s1", 40, 200, WP),
    _W("halo", 64, 16, False, "k3s1", 64, 8, WH),
    _W("halo", 64, 32, False, "k3s1", 40, 24, WH),
    _W("halo", 64, 64, False, "k3s1", 64, 40, WH),
    _W("halo", 64, 128, False, "k3s1", 40, 200, WH),
]

# weight-gradient kernels the dispatch instantiates for no reachable launch, and why (none at present)
WGRAD_UNREACHABLE = {}
