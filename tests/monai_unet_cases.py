"""The launches of build_unet (3dunetcnn_b200/csrc/plan.cu, MONAI UNet) restated once, in plan_launches.py's Launch records, and
the configurations the host tests hold to the library's MAC count, parameter spec and convolution routes.

A MONAI Convolution is its conv (k3s1 / k3s2; transposed: LAYER_CONVT_OP1, a k3s1 conv over the zero-inserted 2n grid whose MACs
count on the input grid, data gradient k3s2 from the 2n grid) then, unless it is conv-only, one norm-apply ("gn", keyed by the
Convolution's prefix).  A ResidualUnit adds its residual conv (k3s2 at stride 2, k1 when only the width changes)."""
from dataclasses import dataclass
from typing import Tuple

from plan_launches import Launch


def unet(n, dims, train=True, input_grad=False, **kw):
    ch = list(kw.get("channels", (16, 32, 64, 128, 256)))
    L, r = len(ch), int(kw.get("num_res_units", 0))
    cin0, cout0 = kw.get("in_channels", 1), kw.get("out_channels", 2)
    ext = [tuple(d >> k for d in dims) for k in range(L)]
    fwd, bwd = [], []

    def conv(pre, ci, co, lvl_in, stride, transposed=False, conv_only=False, first=False):
        key = pre + ".conv.weight"
        if transposed:
            e_out = ext[lvl_in - 1]
            fwd.append(Launch("fwd", key, n, ci, e_out, "k3s1", co, macs_div=8))
            bwd.append(Launch("wgrad", key, n, ci, e_out, "k3s1", co, macs_div=8))
            bwd.append(Launch("dgrad", key, n, co, ext[lvl_in], "k3s2", ci))
        else:
            e_out = ext[lvl_in + (stride == 2)]
            op = "k3s2" if stride == 2 else "k3s1"
            fwd.append(Launch("fwd", key, n, ci, e_out, op, co))
            bwd.append(Launch("wgrad", key, n, ci, e_out, op, co))
            if not first or input_grad:
                bwd.append(Launch("dgrad", key, n, co, ext[lvl_in], "class1" if stride == 2 else "k3s1", ci, reads_input=first))
        if not conv_only:
            fwd.append(Launch("gn", pre, n, co, e_out))

    def down(pre, ci, co, lvl, stride, first=False):
        if r == 0:
            return conv(pre, ci, co, lvl, stride, first=first)
        if stride != 1 or ci != co:
            key = pre + ".residual.weight"
            e_out = ext[lvl + (stride == 2)]
            op = "k3s2" if stride == 2 else "k1"
            fwd.append(Launch("fwd", key, n, ci, e_out, op, co))
            bwd.append(Launch("wgrad", key, n, ci, e_out, op, co))
            if not first or input_grad:
                bwd.append(Launch("dgrad", key, n, co, ext[lvl], "class1" if stride == 2 else "k1", ci, reads_input=first))
        for u in range(r):
            conv("%s.conv.unit%d" % (pre, u), ci if u == 0 else co, co, lvl if u == 0 else lvl + (stride == 2),
                 stride if u == 0 else 1, first=first and u == 0)

    def up(pre, upc, outc, lvl, top):
        if r == 0:
            return conv(pre, upc, outc, lvl + 1, 2, transposed=True, conv_only=top)
        conv(pre + ".0", upc, outc, lvl + 1, 2, transposed=True)
        conv(pre + ".1.conv.unit0", outc, outc, lvl, 1, conv_only=top)

    def level(i):
        pre = "model." + "1.submodule." * i
        down(pre + "0", cin0 if i == 0 else ch[i - 1], ch[i], i, 2, first=i == 0)
        if i + 2 < L:
            level(i + 1)
            upc = 2 * ch[i]
        else:
            down(pre + "1.submodule", ch[i], ch[L - 1], i + 1, 1)
            upc = ch[i] + ch[L - 1]
        up(pre + "2", upc, cout0 if i == 0 else ch[i - 1], i, i == 0)
    level(0)
    return fwd + (bwd if train else [])


@dataclass(frozen=True)
class Config:
    name: str
    kw: dict
    n: int
    dims: Tuple[int, int, int]
    train: bool = True
    input_grad: bool = False

    def launches(self):
        return unet(self.n, self.dims, self.train, self.input_grad, **self.kw)


SPLEEN = dict(in_channels=1, out_channels=2, channels=(16, 32, 64, 128, 256), strides=(2, 2, 2, 2), num_res_units=2)
BRATS = dict(SPLEEN, in_channels=4, out_channels=3)
# the two workloads tools/monai_unet_bench.py times, their forward-only and input-gradient plans, and the small networks of
# tests/test_gpu_monai_unet.py (no residual units: the conv-only transposed top layer; an equal-width bottom: identity residual)
CONFIGS = [Config("spleen", SPLEEN, 4, (96, 96, 96)), Config("spleen-infer", SPLEEN, 4, (96, 96, 96), train=False),
           Config("brats", BRATS, 2, (128, 128, 128), input_grad=True),
           Config("r0-prelu", dict(in_channels=1, out_channels=2, channels=(8, 16, 32), strides=(2, 2)), 2, (32, 32, 32),
                  input_grad=True),
           Config("r0-affine-16in", dict(in_channels=16, out_channels=16, channels=(16, 32, 64), strides=(2, 2), bias=False,
                                          norm=("instance", {"affine": True}), act="relu"), 1, (32, 48, 64), input_grad=True),
           Config("r1-equal-bottom", dict(in_channels=4, out_channels=2, channels=(16, 16), strides=(2,), num_res_units=1), 1,
                  (32, 32, 32), input_grad=True)]
