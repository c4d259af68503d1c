"""ctypes binding of libb200unet.so (C ABI declared in include/b200unet.h).

PyTorch is used for device memory and streams only: every call passes raw device pointers and the current CUDA
stream.  A non-zero status raises ``RuntimeError`` with the library's message -- there is no CPU or PyTorch
fallback; a missing library raises at import of the op, loudly.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200UNET_LIB: load a differently-built copy of the library (A/B runs of compile-time kernel variants: `make BUILD=... OUT=... EXTRA=-D...` in csrc/)
LIB_PATH = os.environ.get("B200UNET_LIB") or os.path.join(_HERE, "libb200unet.so")
CSRC = os.path.join(_HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include", "b200unet.h")
INCLUDE_DIAG = os.path.join(os.path.dirname(_HERE), "include", "b200unet_diag.h")


class Tensor5(C.Structure):
    """``b200unet_tensor``: NDHWC bf16 view (hi [+ lo])."""
    _fields_ = [("hi", C.c_void_p), ("lo", C.c_void_p), ("n", C.c_int32), ("d", C.c_int32), ("h", C.c_int32),
                ("w", C.c_int32), ("c", C.c_int32), ("ld", C.c_int32)]


class ConvDesc(C.Structure):
    _fields_ = [("x", Tensor5 * 2), ("w_hi", C.c_void_p * 2), ("w_lo", C.c_void_p * 2), ("ksz", C.c_int32 * 2),
                ("stride", C.c_int32 * 2), ("cip", C.c_int32 * 2), ("nsrc", C.c_int32), ("cop", C.c_int32),
                ("out", Tensor5), ("res", C.POINTER(Tensor5)), ("scale", C.c_void_p), ("stats", C.c_void_p),
                ("stats_ld", C.c_int32), ("mode", C.c_int32), ("gn_x", C.POINTER(Tensor5)), ("coef", C.c_void_p),
                ("coef_ld", C.c_int32), ("slope", C.c_float), ("bstats", C.c_void_p), ("cls_mode", C.c_int32)]


class DiagExt(C.Structure):
    """``b200unet_diag_ext``: bias, zeroed high boundary and visible extents (include/b200unet_diag.h)."""
    _fields_ = [("bias", C.c_void_p), ("zero_last", C.c_int32), ("x_vis", (C.c_int32 * 3) * 2), ("a_vis", C.c_int32 * 3),
                ("dy_vis", C.c_int32 * 3), ("max_ctas", C.c_int32)]


class ConvRoute(C.Structure):
    _fields_ = [("kind", C.c_int32), ("bn", C.c_int32), ("kc", C.c_int32), ("kchunks", C.c_int32 * 2), ("npass", C.c_int32),
                ("cls_pair", C.c_int32), ("tw", C.c_int32), ("th", C.c_int32), ("td", C.c_int32), ("grid", C.c_int32 * 3),
                ("stages", C.c_int32), ("blocks_per_sm", C.c_int32), ("smem_bytes", C.c_int32)]


class WgradRoute(C.Structure):
    _fields_ = [("kind", C.c_int32), ("ci8", C.c_int32), ("cb", C.c_int32), ("bn", C.c_int32), ("qt", C.c_int32),
                ("groups", C.c_int32), ("cotiles", C.c_int32), ("kblocks", C.c_int32), ("splits", C.c_int32), ("npass", C.c_int32),
                ("tw", C.c_int32), ("th", C.c_int32), ("td", C.c_int32), ("part_bytes", C.c_int64)]


CONV_KINDS = ("tap", "halo", "class1", "class2")     # b200unet_conv_route.kind
WGRAD_KINDS = ("simt", "tap", "halo")               # b200unet_wgrad_route.kind


class DiceCEDesc(C.Structure):
    """``b200unet_dice_ce_desc``: options of the Dice + cross-entropy criterion."""
    _fields_ = [("act", C.c_int32), ("target_kind", C.c_int32), ("include_background", C.c_int32), ("squared_pred", C.c_int32),
                ("jaccard", C.c_int32), ("batch", C.c_int32), ("reduction", C.c_int32), ("smooth_nr", C.c_float),
                ("smooth_dr", C.c_float), ("lambda_dice", C.c_float), ("lambda_ce", C.c_float)]


class NetDesc(C.Structure):
    _fields_ = [("n_features", C.c_int32), ("n_outputs", C.c_int32), ("base_width", C.c_int32),
                ("n_levels", C.c_int32), ("encoder_blocks", C.c_int32 * 8), ("decoder_blocks", C.c_int32 * 8),
                ("feature_dilation", C.c_int32), ("norm_groups", C.c_int32),
                ("use_transposed_convolutions", C.c_int32), ("activation", C.c_int32),
                ("split_precision", C.c_int32), ("batch", C.c_int32), ("depth", C.c_int32), ("height", C.c_int32),
                ("width", C.c_int32), ("arch", C.c_int32), ("filters", C.c_int32 * 8), ("act_slope", C.c_float),
                ("deterministic", C.c_int32), ("inference_only", C.c_int32), ("input_grad", C.c_int32)]


def build_library(force: bool = False, verbose: bool = False) -> str:
    """Compile libb200unet.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
    if os.environ.get("B200UNET_LIB"):
        return LIB_PATH                       # an explicitly chosen variant is never rebuilt behind the caller's back
    if os.path.exists(LIB_PATH) and not force:
        src_m = max(os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC)
                    if f.endswith((".cu", ".cuh", ".h")) or f == "Makefile")
        src_m = max(src_m, os.path.getmtime(INCLUDE), os.path.getmtime(INCLUDE_DIAG))
        if os.path.getmtime(LIB_PATH) >= src_m:
            return LIB_PATH
    cmd = ["make", "-C", CSRC, "-j8"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        print(res.stdout[-4000:])
        print(res.stderr[-8000:])
    if res.returncode != 0:
        raise RuntimeError("building libb200unet.so failed (nvcc): see output above")
    return LIB_PATH


_lib = None

_SIGS = {
    "b200unet_version": (C.c_int, []),
    "b200unet_last_error": (C.c_char_p, []),
    "b200unet_ncdhw_to_ndhwc": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(Tensor5), C.c_void_p]),
    "b200unet_ndhwc_to_ncdhw": (C.c_int, [C.POINTER(Tensor5), C.c_int, C.c_void_p, C.c_void_p]),
    "b200unet_pack_weights": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                        C.c_void_p, C.c_void_p]),
    "b200unet_unpack_wgrad": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                        C.c_void_p]),
    "b200unet_conv3d": (C.c_int, [C.POINTER(ConvDesc), C.c_void_p]),
    "b200unet_conv3d_wgrad": (C.c_int, [C.POINTER(Tensor5), C.POINTER(Tensor5), C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.c_void_p, C.c_void_p]),
    "b200unet_gn_apply": (C.c_int, [C.POINTER(Tensor5), C.POINTER(Tensor5), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                    C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    "b200unet_gn_bwd_finalize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                           C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200unet_gn_bwd": (C.c_int, [C.POINTER(Tensor5), C.POINTER(Tensor5), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                  C.c_void_p, C.c_void_p, C.POINTER(Tensor5), C.POINTER(Tensor5), C.POINTER(Tensor5), C.c_void_p]),
    "b200unet_upsample2x_fwd": (C.c_int, [C.POINTER(Tensor5), C.POINTER(Tensor5), C.c_void_p, C.c_int, C.c_void_p]),
    "b200unet_upsample2x_bwd": (C.c_int, [C.POINTER(Tensor5), C.POINTER(Tensor5), C.c_void_p]),
    "b200unet_zero_insert": (C.c_int, [C.POINTER(Tensor5), C.POINTER(Tensor5), C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200unet_head_fwd": (C.c_int, [C.POINTER(Tensor5), C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "b200unet_head_bwd_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "b200unet_head_bwd": (C.c_int, [C.POINTER(Tensor5), C.c_void_p, C.c_int, C.c_void_p, C.POINTER(Tensor5),
                                    C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200unet_dice_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_float,
                                    C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200unet_dice_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_float,
                                    C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200unet_dice_ce_scratch_bytes": (C.c_size_t, [C.POINTER(DiceCEDesc), C.c_int, C.c_int, C.c_int64]),
    "b200unet_dice_ce_fwd": (C.c_int, [C.POINTER(DiceCEDesc), C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_void_p,
                                       C.c_void_p, C.c_void_p]),
    "b200unet_dice_ce_bwd": (C.c_int, [C.POINTER(DiceCEDesc), C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200unet_act_bwd": (C.c_int, [C.POINTER(Tensor5), C.POINTER(Tensor5), C.POINTER(Tensor5), C.c_void_p, C.c_float,
                                   C.POINTER(Tensor5), C.c_void_p, C.c_int, C.c_void_p]),
    "b200unet_tiles_gather": (C.c_int, [C.c_void_p] + [C.c_int] * 5 + [C.POINTER(C.c_int32), C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.c_void_p, C.c_void_p]),
    "b200unet_tiles_scatter": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200unet_tiles_count": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200unet_tiles_normalize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p]),
    "b200unet_one_hot": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.POINTER(C.c_float), C.POINTER(C.c_int32), C.c_int, C.c_int,
                                   C.c_void_p, C.c_void_p]),
    "b200unet_zscore": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200unet_label_map": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.POINTER(C.c_int32), C.c_int, C.c_float, C.c_int, C.c_int,
                                     C.c_void_p, C.c_void_p]),
    "b200unet_cc_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "b200unet_cc_label": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p]),
    "b200unet_cc_sort_by_size": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "b200unet_plan_create": (C.c_int, [C.POINTER(NetDesc), C.POINTER(C.c_void_p)]),
    "b200unet_plan_destroy": (None, [C.c_void_p]),
    "b200unet_plan_num_params": (C.c_int, [C.c_void_p]),
    "b200unet_plan_param_info": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int64), C.c_char_p, C.c_int]),
    "b200unet_plan_workspace_bytes": (C.c_size_t, [C.c_void_p]),
    "b200unet_plan_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200unet_plan_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                         C.c_void_p, C.c_void_p]),
    "b200unet_plan_input_grad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200unet_plan_backward_parts": (C.c_int, [C.c_void_p]),
    "b200unet_plan_param_backward_part": (C.c_int, [C.c_void_p, C.c_int]),
    "b200unet_plan_backward_part": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                              C.c_void_p, C.c_void_p]),
    "b200unet_plan_last_launches": (C.c_int, [C.c_void_p]),
    "b200unet_plan_algorithmic_macs": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.c_int]),
    "b200unet_plan_profile_begin": (C.c_int, [C.c_void_p, C.c_int]),
    "b200unet_plan_profile_end": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int64), C.c_int]),
    "b200unet_plan_profile_dump": (C.c_int, [C.c_void_p, C.c_char_p]),
}

# entry points outside the product header (include/b200unet_diag.h), bound like _SIGS
_WG_ARGS = [C.POINTER(Tensor5), C.POINTER(Tensor5), C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(DiagExt)]
_DIAG_SIGS = {
    "b200unet_diag_conv3d_route": (C.c_int, [C.POINTER(ConvDesc), C.POINTER(DiagExt), C.POINTER(ConvRoute)]),
    "b200unet_diag_wgrad_route": (C.c_int, _WG_ARGS + [C.c_int, C.c_int, C.POINTER(WgradRoute)]),
    "b200unet_diag_wgrad_partial_bytes": (C.c_size_t, _WG_ARGS + [C.c_int]),
    "b200unet_diag_conv3d_ex": (C.c_int, [C.POINTER(ConvDesc), C.POINTER(DiagExt), C.c_void_p]),
    "b200unet_diag_wgrad_ex": (C.c_int, _WG_ARGS + [C.c_void_p, C.c_size_t, C.POINTER(C.c_int), C.c_void_p, C.c_void_p]),
    "b200unet_diag_bias_grad": (C.c_int, [C.POINTER(Tensor5), C.POINTER(DiagExt), C.c_void_p, C.c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_SIGS)


def load_library():
    """dlopen the in-tree library (building it first if sources are newer) and set signatures."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        build_library()
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in list(_SIGS.items()) + list(_DIAG_SIGS.items()):
        fn = getattr(lib, name)  # AttributeError if the symbol is missing: fail loudly
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int, what: str = "") -> None:
    if status != 0:
        msg = load_library().b200unet_last_error()
        raise RuntimeError("libb200unet %s failed (status %d): %s" % (what, status, msg.decode() if msg else "?"))


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------ tensor helpers
class Act:
    """NDHWC bf16 activation (hi [+ lo]) living in torch tensors; ``c`` visible channels out of ``ld``."""

    def __init__(self, hi: torch.Tensor, lo: Optional[torch.Tensor] = None, c0: int = 0, c: Optional[int] = None):
        assert hi.dtype == torch.bfloat16 and hi.dim() == 5 and hi.is_contiguous()
        self.hi, self.lo = hi, lo
        self.n, self.d, self.h, self.w, self.ld = hi.shape
        self.c0 = c0
        self.c = self.ld - c0 if c is None else c

    @staticmethod
    def empty(n, d, h, w, c, split=False, device="cuda", zero=False):
        mk = torch.zeros if zero else torch.empty
        hi = mk((n, d, h, w, c), dtype=torch.bfloat16, device=device)
        lo = mk((n, d, h, w, c), dtype=torch.bfloat16, device=device) if split else None
        return Act(hi, lo)

    @staticmethod
    def from_ncdhw(x: torch.Tensor, split=False, pad_to: int = 8):
        """fp32 NCDHW torch tensor -> Act (through the library's converter)."""
        n, c, d, h, w = x.shape
        cp = (c + pad_to - 1) // pad_to * pad_to
        a = Act.empty(n, d, h, w, cp, split=split, device=x.device)
        lib = load_library()
        x = x.contiguous().float()
        check(lib.b200unet_ncdhw_to_ndhwc(x.data_ptr(), c, C.byref(a.ct()), stream_ptr()), "ncdhw_to_ndhwc")
        return a

    def slice(self, c0, c):
        return Act(self.hi, self.lo, self.c0 + c0, c)

    def ct(self) -> Tensor5:
        t = Tensor5()
        t.hi = self.hi.data_ptr() + 2 * self.c0
        t.lo = (self.lo.data_ptr() + 2 * self.c0) if self.lo is not None else None
        t.n, t.d, t.h, t.w, t.c, t.ld = self.n, self.d, self.h, self.w, self.c, self.ld
        return t

    def to_ncdhw(self, c_real: Optional[int] = None) -> torch.Tensor:
        c_real = self.c if c_real is None else c_real
        y = torch.empty((self.n, c_real, self.d, self.h, self.w), dtype=torch.float32, device=self.hi.device)
        check(load_library().b200unet_ndhwc_to_ncdhw(C.byref(self.ct()), c_real, y.data_ptr(), stream_ptr()),
              "ndhwc_to_ncdhw")
        return y

    def value(self) -> torch.Tensor:
        """fp32 NDHWC value of the visible slice (torch math; for tests)."""
        v = self.hi[..., self.c0:self.c0 + self.c].float()
        if self.lo is not None:
            v = v + self.lo[..., self.c0:self.c0 + self.c].float()
        return v


def pack_weights(w: torch.Tensor, mode: int = 0, split: bool = False, cop: Optional[int] = None,
                 cip: Optional[int] = None):
    """torch conv weight -> packed bf16 GEMM operand(s).  Returns (hi, lo|None, cop, cip, taps)."""
    w = w.contiguous().float()
    if mode >= 2:                                   # ConvTranspose3d weight [Ci][Co][k^3]
        ci, co = w.shape[0], w.shape[1]
    else:
        co, ci = w.shape[0], w.shape[1]
    taps = int(w.shape[2] * w.shape[3] * w.shape[4])
    cop = (co + 7) // 8 * 8 if cop is None else cop
    cip = (ci + 7) // 8 * 8 if cip is None else cip
    shape = (taps, cip, cop) if mode in (1, 3) else (taps, cop, cip)
    hi = torch.empty(shape, dtype=torch.bfloat16, device=w.device)
    lo = torch.empty(shape, dtype=torch.bfloat16, device=w.device) if split else None
    check(load_library().b200unet_pack_weights(w.data_ptr(), co, ci, cop, cip, taps, mode, hi.data_ptr(),
                                               lo.data_ptr() if split else None, stream_ptr()), "pack_weights")
    return hi, lo, cop, cip, taps


def conv3d(x: Act, w_hi, w_lo, ksz: int, stride: int, out: Act, cop: int, cip: int, *, x2: Optional[Act] = None,
           w2_hi=None, w2_lo=None, cip2: int = 0, res: Optional[Act] = None, scale: Optional[torch.Tensor] = None,
           stats: Optional[torch.Tensor] = None, stats_ld: int = 0, mode: int = 0, gn_x: Optional[Act] = None,
           coef: Optional[torch.Tensor] = None, coef_ld: int = 0, slope: float = 0.0,
           bstats: Optional[torch.Tensor] = None, cls_mode: int = 0) -> None:
    d, keep = conv_desc(**locals())
    check(load_library().b200unet_conv3d(C.byref(d), stream_ptr()), "conv3d")


def conv_desc(x: Act, w_hi, w_lo, ksz: int, stride: int, out: Act, cop: int, cip: int, *, x2: Optional[Act] = None,
              w2_hi=None, w2_lo=None, cip2: int = 0, res: Optional[Act] = None, scale: Optional[torch.Tensor] = None,
              stats: Optional[torch.Tensor] = None, stats_ld: int = 0, mode: int = 0, gn_x: Optional[Act] = None,
              coef: Optional[torch.Tensor] = None, coef_ld: int = 0, slope: float = 0.0,
              bstats: Optional[torch.Tensor] = None, cls_mode: int = 0):
    """``b200unet_conv_desc`` of a conv3d call, and the structures it points to (keep them alive while it is used)"""
    d = ConvDesc()
    d.x[0] = x.ct()
    d.w_hi[0] = w_hi.data_ptr()
    d.w_lo[0] = w_lo.data_ptr() if w_lo is not None else None
    d.ksz[0], d.stride[0], d.cip[0] = ksz, stride, cip
    d.nsrc = 1
    if x2 is not None:
        d.x[1] = x2.ct()
        d.w_hi[1] = w2_hi.data_ptr()
        d.w_lo[1] = w2_lo.data_ptr() if w2_lo is not None else None
        d.ksz[1], d.stride[1], d.cip[1] = 1, 1, cip2
        d.nsrc = 2
    d.cop = cop
    d.out = out.ct()
    keep = []
    if res is not None:
        r = res.ct(); keep.append(r)
        d.res = C.pointer(r)
    d.scale = scale.data_ptr() if scale is not None else None
    d.stats = stats.data_ptr() if stats is not None else None
    d.stats_ld = stats_ld
    d.mode = mode
    if gn_x is not None:
        g = gn_x.ct(); keep.append(g)
        d.gn_x = C.pointer(g)
    d.coef = coef.data_ptr() if coef is not None else None
    d.coef_ld = coef_ld
    d.slope = slope
    d.bstats = bstats.data_ptr() if bstats is not None else None
    d.cls_mode = cls_mode
    return d, keep


def diag_ext(bias: Optional[torch.Tensor] = None, zero_last: bool = False, x_vis=None, a_vis=None, dy_vis=None,
             max_ctas: int = 0) -> DiagExt:
    """``b200unet_diag_ext``; each *_vis is a (d, h, w) triple (x_vis: one per source), 0 = the full extent; max_ctas > 0 caps
    the CTAs per N tile of the persistent halo kernel"""
    e = DiagExt()
    e.max_ctas = max_ctas
    e.bias = _p(bias)
    e.zero_last = int(bool(zero_last))
    for s, v in enumerate(x_vis or ()):
        e.x_vis[s][:] = list(v)
    if a_vis is not None:
        e.a_vis[:] = list(a_vis)
    if dy_vis is not None:
        e.dy_vis[:] = list(dy_vis)
    return e


def _route_dict(r) -> dict:
    out = {}
    for name, _ in r._fields_:
        v = getattr(r, name)
        out[name] = tuple(v) if not isinstance(v, int) else v
    return out


def conv3d_route(*args, ext: Optional[DiagExt] = None, **kw) -> dict:
    """the kernel route b200unet_conv3d takes for these conv3d arguments (host-only query; RuntimeError if it refuses them).
    ``kind`` is one of CONV_KINDS."""
    d, keep = conv_desc(*args, **kw)
    r = ConvRoute()
    check(load_library().b200unet_diag_conv3d_route(C.byref(d), C.byref(ext) if ext is not None else None, C.byref(r)),
          "diag_conv3d_route")
    out = _route_dict(r)
    out["kind"] = CONV_KINDS[r.kind]
    return out


def conv3d_ex(*args, ext: Optional[DiagExt] = None, **kw) -> None:
    """conv3d with the options only the plans set (bias, zero_last, visible source extents)"""
    d, keep = conv_desc(*args, **kw)
    check(load_library().b200unet_diag_conv3d_ex(C.byref(d), C.byref(ext) if ext is not None else None, stream_ptr()),
          "diag_conv3d_ex")


def wgrad_route(a: Act, dy: Act, ksz: int, stride: int, cip: int, cop: int, *, deterministic: bool = False, num_sms: int = 132,
                ext: Optional[DiagExt] = None) -> dict:
    """the kernel route of a weight gradient on a device with num_sms SMs (host-only query).  ``kind`` is one of WGRAD_KINDS."""
    r = WgradRoute()
    check(load_library().b200unet_diag_wgrad_route(C.byref(a.ct()), C.byref(dy.ct()), ksz, stride, cip, cop,
                                                   C.byref(ext) if ext is not None else None, int(bool(deterministic)), num_sms,
                                                   C.byref(r)), "diag_wgrad_route")
    out = _route_dict(r)
    out["kind"] = WGRAD_KINDS[r.kind]
    return out


def wgrad_partial_bytes(a: Act, dy: Act, ksz: int, stride: int, cip: int, cop: int, num_sms: int = 132,
                        ext: Optional[DiagExt] = None) -> int:
    return int(load_library().b200unet_diag_wgrad_partial_bytes(C.byref(a.ct()), C.byref(dy.ct()), ksz, stride, cip, cop,
                                                                C.byref(ext) if ext is not None else None, num_sms))


def wgrad_ex(a: Act, dy: Act, ksz: int, stride: int, cip: int, cop: int, dw: torch.Tensor, *, part: Optional[torch.Tensor] = None,
             part_bytes: Optional[int] = None, ext: Optional[DiagExt] = None) -> int:
    """the weight gradient as the plans run it: atomics into dw (part None), or the deterministic partial sums in part
    followed by their fixed-order reduction into dw.  Returns the number of partial slots written (0 with atomics)."""
    splits = C.c_int(0)
    nbytes = (part.numel() * part.element_size() if part is not None else 0) if part_bytes is None else part_bytes
    check(load_library().b200unet_diag_wgrad_ex(C.byref(a.ct()), C.byref(dy.ct()), ksz, stride, cip, cop,
                                                C.byref(ext) if ext is not None else None, _p(part), nbytes, C.byref(splits),
                                                dw.data_ptr(), stream_ptr()), "diag_wgrad_ex")
    return splits.value


def bias_grad(dy: Act, dbias: torch.Tensor, ext: Optional[DiagExt] = None) -> None:
    """dbias = sum of dy over its visible voxels (ext.dy_vis)"""
    check(load_library().b200unet_diag_bias_grad(C.byref(dy.ct()), C.byref(ext) if ext is not None else None, dbias.data_ptr(),
                                                 stream_ptr()), "diag_bias_grad")


def conv3d_wgrad(a: Act, dy: Act, ksz: int, stride: int, cip: int, cop: int, dw: torch.Tensor) -> None:
    check(load_library().b200unet_conv3d_wgrad(C.byref(a.ct()), C.byref(dy.ct()), ksz, stride, cip, cop, dw.data_ptr(),
                                               stream_ptr()), "conv3d_wgrad")


def _p(t: Optional[torch.Tensor]):
    return t.data_ptr() if t is not None else None


def gn_apply(x: Act, y: Act, stats, gamma, beta, c, groups, coef, eps=1e-5, slope=0.0) -> None:
    """y = act(GroupNorm(x)) from the fp64 (sum, sumsq) statistics [n][x.c][2] of the c real channels; writes coef [n][x.c][4]"""
    check(load_library().b200unet_gn_apply(C.byref(x.ct()), C.byref(y.ct()), stats.data_ptr(), _p(gamma), _p(beta), c, groups,
                                           eps, slope, coef.data_ptr(), stream_ptr()), "gn_apply")


def gn_bwd_finalize(bstats, coef, gamma, n, c, c_ld, groups, spatial, coef2, dgamma, dbeta) -> None:
    check(load_library().b200unet_gn_bwd_finalize(bstats.data_ptr(), coef.data_ptr(), _p(gamma), n, c, c_ld, groups,
                                                  spatial, coef2.data_ptr(), _p(dgamma), _p(dbeta), stream_ptr()),
          "gn_bwd_finalize")


def gn_bwd(dz: Act, x: Act, coef, bstats, gamma, c, groups, dx: Act, dgamma=None, dbeta=None, add1: Optional[Act] = None,
           add2: Optional[Act] = None) -> None:
    """dx (+ add1 + add2) and dgamma / dbeta from the backward statistics bstats [n][x.c][2] = (sum dz, sum dz * xhat)"""
    a1 = add1.ct() if add1 is not None else None
    a2 = add2.ct() if add2 is not None else None
    check(load_library().b200unet_gn_bwd(C.byref(dz.ct()), C.byref(x.ct()), coef.data_ptr(), bstats.data_ptr(), _p(gamma), c,
                                         groups, _p(dgamma), _p(dbeta), C.byref(a1) if a1 is not None else None,
                                         C.byref(a2) if a2 is not None else None, C.byref(dx.ct()), stream_ptr()), "gn_bwd")


def upsample2x_fwd(x: Act, y: Act, stats=None, stats_ld=0) -> None:
    check(load_library().b200unet_upsample2x_fwd(C.byref(x.ct()), C.byref(y.ct()), _p(stats), stats_ld, stream_ptr()),
          "upsample2x_fwd")


def upsample2x_bwd(dy: Act, dx: Act) -> None:
    check(load_library().b200unet_upsample2x_bwd(C.byref(dy.ct()), C.byref(dx.ct()), stream_ptr()), "upsample2x_bwd")


def zero_insert(x: Act, z: Act, od=0, oh=0, ow=0) -> None:
    check(load_library().b200unet_zero_insert(C.byref(x.ct()), C.byref(z.ct()), od, oh, ow, stream_ptr()),
          "zero_insert")


def head_fwd(x: Act, w: torch.Tensor, n_out: int, act: int, logits: torch.Tensor) -> None:
    check(load_library().b200unet_head_fwd(C.byref(x.ct()), w.data_ptr(), n_out, act, logits.data_ptr(), stream_ptr()),
          "head_fwd")


def head_bwd(x: Act, w, n_out, dlogits, dx: Act, dw) -> None:
    lib = load_library()
    scratch = torch.empty(int(lib.b200unet_head_bwd_scratch_bytes(n_out, x.c)), dtype=torch.uint8, device=x.hi.device)
    check(lib.b200unet_head_bwd(C.byref(x.ct()), w.data_ptr(), n_out, dlogits.data_ptr(), C.byref(dx.ct()),
                                dw.data_ptr(), scratch.data_ptr(), stream_ptr()), "head_bwd")


def dice_flags(sigmoid=True, squared_pred=False, jaccard=False, batch=False, include_background=True,
               reduction="mean", float_target=False) -> int:
    if reduction not in ("mean", "sum"):
        raise ValueError("fused Dice supports reduction 'mean' or 'sum', got %r" % (reduction,))
    return (int(bool(sigmoid)) | (int(bool(squared_pred)) << 1) | (int(bool(jaccard)) << 2) | (int(bool(batch)) << 3)
            | (int(not include_background) << 4) | (int(reduction == "sum") << 5) | (int(bool(float_target)) << 6))


def dice_fwd(logits, target, flags, nr, dr, sums, loss) -> None:
    n, c = logits.shape[:2]
    s = logits[0, 0].numel()
    check(load_library().b200unet_dice_fwd(logits.data_ptr(), target.data_ptr(), n, c, s, flags, nr, dr,
                                           sums.data_ptr(), loss.data_ptr(), stream_ptr()), "dice_fwd")


def dice_bwd(logits, target, flags, nr, dr, sums, grad_out, dlogits) -> None:
    n, c = logits.shape[:2]
    s = logits[0, 0].numel()
    check(load_library().b200unet_dice_bwd(logits.data_ptr(), target.data_ptr(), n, c, s, flags, nr, dr,
                                           sums.data_ptr(), grad_out.data_ptr(), dlogits.data_ptr(), stream_ptr()),
          "dice_bwd")


# b200unet_dice_ce_desc.target_kind of each target form
DICE_CE_TARGETS = {"label_u8": 0, "label_i64": 1, "onehot_u8": 2, "soft_f32": 3}
_DICE_CE_ACTS = {None: 0, "sigmoid": 1, "softmax": 2}


def dice_ce_desc(act=None, target_kind=0, include_background=True, squared_pred=False, jaccard=False, batch=False,
                 reduction="mean", smooth_nr=1e-5, smooth_dr=1e-5, lambda_dice=1.0, lambda_ce=1.0) -> DiceCEDesc:
    if reduction not in ("mean", "sum"):
        raise ValueError("fused DiceCE supports reduction 'mean' or 'sum', got %r" % (reduction,))
    d = DiceCEDesc()
    d.act, d.target_kind = _DICE_CE_ACTS[act], int(target_kind)
    d.include_background, d.squared_pred, d.jaccard, d.batch = (int(bool(v)) for v in (include_background, squared_pred, jaccard, batch))
    d.reduction = int(reduction == "sum")
    d.smooth_nr, d.smooth_dr, d.lambda_dice, d.lambda_ce = float(smooth_nr), float(smooth_dr), float(lambda_dice), float(lambda_ce)
    return d


def _nc_s(logits):
    return logits.shape[0], logits.shape[1], logits[0, 0].numel()


def dice_ce_scratch_bytes(desc: DiceCEDesc, n: int, c: int, s: int) -> int:
    lib = load_library()
    b = int(lib.b200unet_dice_ce_scratch_bytes(C.byref(desc), n, c, s))
    if b == 0:
        msg = lib.b200unet_last_error()
        raise RuntimeError("libb200unet dice_ce_scratch_bytes rejected n=%d c=%d spatial=%d: %s" % (n, c, s, msg.decode() if msg else "?"))
    return b


def cc_scratch_bytes(nvol: int, d: int, h: int, w: int) -> int:
    lib = load_library()
    b = int(lib.b200unet_cc_scratch_bytes(nvol, d, h, w))
    if b == 0:
        msg = lib.b200unet_last_error()
        raise RuntimeError("libb200unet cc_scratch_bytes rejected %d x %d x %d x %d: %s" % (nvol, d, h, w, msg.decode() if msg else "?"))
    return b


def _need_c_order(**tensors) -> None:
    for name, t in tensors.items():
        if not t.is_contiguous():
            raise ValueError("%s must be contiguous (C order): the kernels read it as a dense [nvol, d, h, w] array" % name)


def cc_label(mask, connectivity, labels, counts, scratch) -> None:
    """mask uint8 [nvol, d, h, w] -> raster-order labels int32 (same shape) and counts int32 [nvol]"""
    _need_c_order(mask=mask, labels=labels)
    nvol, d, h, w = mask.shape
    check(load_library().b200unet_cc_label(mask.data_ptr(), nvol, d, h, w, connectivity, labels.data_ptr(), counts.data_ptr(),
                                           scratch.data_ptr(), stream_ptr()), "cc_label")


def cc_sort_by_size(labels, max_count, scratch) -> None:
    _need_c_order(labels=labels)
    nvol, d, h, w = labels.shape
    check(load_library().b200unet_cc_sort_by_size(labels.data_ptr(), nvol, d, h, w, max_count, scratch.data_ptr(), stream_ptr()),
          "cc_sort_by_size")


def dice_ce_fwd(desc: DiceCEDesc, logits, target, scratch, loss) -> None:
    n, c, s = _nc_s(logits)
    check(load_library().b200unet_dice_ce_fwd(C.byref(desc), logits.data_ptr(), target.data_ptr(), n, c, s, scratch.data_ptr(),
                                              loss.data_ptr(), stream_ptr()), "dice_ce_fwd")


def dice_ce_bwd(desc: DiceCEDesc, logits, target, scratch, grad_out, dlogits) -> None:
    n, c, s = _nc_s(logits)
    check(load_library().b200unet_dice_ce_bwd(C.byref(desc), logits.data_ptr(), target.data_ptr(), n, c, s, scratch.data_ptr(),
                                              grad_out.data_ptr(), dlogits.data_ptr(), stream_ptr()), "dice_ce_bwd")
