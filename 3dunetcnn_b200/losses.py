"""Fused Dice and Dice + cross-entropy criteria -- the classes ``load_criterion`` finds first.

The reference resolves ``config["loss"]["name"]`` in ``unet3d.losses`` before ``torch.nn`` and ``monai.losses``
(/root/reference/unet3d/scripts/script_utils.py:64-73; the shipped module is an empty hook,
unet3d/losses/losses.py:1-3), so a class named ``DiceLoss`` placed here takes over
``{"name": "DiceLoss", "include_background": true, "sigmoid": true}``
(examples/brats2020/brats2020_config.json:112-116) with MONAI's kwarg names.  Forward and backward are the
hand-written kernels ``b200unet_dice_fwd`` / ``b200unet_dice_bwd``; targets stay uint8 in HBM.  ``DiceCELoss`` takes over
``{"name": "DiceCELoss", "softmax": true, "to_onehot_y": true}`` the same way, on ``b200unet_dice_ce_fwd`` / ``_bwd``: it reads
a one-channel label map (or a C-channel target) and adds cross-entropy to a softmax Dice.  ``TverskyLoss``,
``GeneralizedDiceLoss``, ``FocalLoss`` and ``DiceFocalLoss`` run on the same entry points with the same target forms: another
overlap of the same per-(n, c) sums, or the focal term in CE's place.  ``HausdorffDTLoss`` and ``LogHausdorffDTLoss`` take the
distance-weighted term in its place, on weights ``b200unet_hausdorff_dt_weight`` computes from exact distance transforms.
"""
from __future__ import annotations

import warnings

import torch
from torch import nn

from . import lib as _lib

_SURFACE_MAX_EXTENT = 256      # B200_SURFACE_MAX_EXTENT: voxels per axis of the distance transforms (HausdorffDTLoss)


class _DiceFunction(torch.autograd.Function):
    """Both criteria: ``fwd`` / ``bwd`` are the pair of entry points (``lib.dice_*`` or ``lib.dice_ce_*``) and ``scratch_len``
    the fp64 scratch they share (the sums, the backward coefficients and any per-block partials; no host synchronisation)."""

    @staticmethod
    def forward(ctx, logits, target, desc, fwd, bwd, scratch_len):
        scratch = torch.empty(scratch_len, dtype=torch.float64, device=logits.device)
        loss = torch.empty((), dtype=torch.float32, device=logits.device)
        fwd(desc, logits, target, scratch, loss)
        ctx.save_for_backward(logits, target, scratch)
        ctx.desc, ctx.bwd = desc, bwd
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        logits, target, scratch = ctx.saved_tensors
        dlogits = torch.empty_like(logits)
        g = grad_out.detach().float().contiguous()
        with torch.cuda.device(logits.device):
            ctx.bwd(ctx.desc, logits, target, scratch, g, dlogits)
        return dlogits, None, None, None, None, None


def _prepare(name: str, output: torch.Tensor, target: torch.Tensor):
    """(contiguous fp32 logits, target with bool as uint8), both plain CUDA tensors"""
    if not output.is_cuda or not target.is_cuda:
        raise RuntimeError("fused %s runs only on CUDA tensors (no CPU fallback)" % name)
    out = output.as_subclass(torch.Tensor) if type(output) is not torch.Tensor else output
    tgt = target.as_subclass(torch.Tensor) if type(target) is not torch.Tensor else target
    return out.contiguous().float(), tgt.to(torch.uint8) if tgt.dtype == torch.bool else tgt


class DiceLoss(nn.Module):
    """MONAI-compatible signature; only the options the kernels implement are accepted (others raise)."""

    def __init__(self, include_background=True, to_onehot_y=False, sigmoid=False, softmax=False, other_act=None,
                 squared_pred=False, jaccard=False, reduction="mean", smooth_nr=1e-5, smooth_dr=1e-5, batch=False,
                 weight=None, **unused):
        super().__init__()
        if softmax or to_onehot_y or other_act is not None or weight is not None:
            raise NotImplementedError("fused DiceLoss: softmax / to_onehot_y / other_act / weight are not implemented")
        if reduction not in ("mean", "sum"):
            raise NotImplementedError("fused DiceLoss: reduction=%r (only 'mean'/'sum')" % (reduction,))
        self._opts = dict(act="sigmoid" if sigmoid else None, include_background=include_background, squared_pred=squared_pred,
                          jaccard=jaccard, batch=batch, reduction=reduction, smooth_nr=smooth_nr, smooth_dr=smooth_dr,
                          lambda_ce=0.0)

    def forward(self, output: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        if output.shape != target.shape:
            raise AssertionError("ground truth has different shape (%s) from input (%s)" % (tuple(target.shape), tuple(output.shape)))
        out, tgt = _prepare("DiceLoss", output, target)
        kinds = _lib.DICE_CE_TARGETS
        if tgt.dtype == torch.uint8:
            kind = kinds["onehot_u8"]
        else:
            # MONAI casts the target to float: soft / interpolated / label-smoothed targets are legal, so any non-uint8
            # target takes the kernels' fp32-target path instead of being truncated to 0/1
            tgt, kind = tgt.float(), kinds["soft_f32"]
        desc = _lib.dice_ce_desc(target_kind=kind, **self._opts)
        n, c = out.shape[:2]
        with torch.cuda.device(out.device):
            return _DiceFunction.apply(out, tgt.contiguous(), desc, _lib.dice_fwd, _lib.dice_bwd, n * c * 5)


class _FusedCriterion(nn.Module):
    """The criteria on ``b200unet_dice_ce_fwd`` / ``_bwd``: MONAI's shape rules for a ``[N,1,...]`` label map (with
    ``to_onehot_y``) or a ``[N,C,...]`` target, and the target forms the kernels read as stored."""

    _name = ""

    def _target_kind(self, c: int, tgt: torch.Tensor):
        """(target as the kernels read it, b200unet_dice_ce_desc.target_kind)"""
        kinds = _lib.DICE_CE_TARGETS
        if c > 1 and tgt.shape[1] == 1:                     # label map
            if tgt.dtype == torch.uint8:
                return tgt, kinds["label_u8"]
            return tgt.long(), kinds["label_i64"]
        if tgt.dtype == torch.uint8:                         # one-hot (or, with C == 1, the single target channel)
            return tgt, kinds["onehot_u8"]
        return tgt.float(), kinds["soft_f32"]

    def _check_shapes(self, input: torch.Tensor, target: torch.Tensor) -> None:
        if input.dim() != target.dim():
            raise ValueError("the number of dimensions for input and target should be the same, got shape %s and %s"
                             % (tuple(input.shape), tuple(target.shape)))
        c, tc = input.shape[1], target.shape[1]
        if tc != 1 and tc != c:
            raise ValueError("number of channels for target is neither 1 nor the same as input, got shape %s and %s"
                             % (tuple(input.shape), tuple(target.shape)))
        if target.shape[0] != input.shape[0] or target.shape[2:] != input.shape[2:]:
            raise ValueError("target shape %s does not match input shape %s" % (tuple(target.shape), tuple(input.shape)))
        if c > 1 and self.to_onehot_y and tc != 1:
            raise ValueError("to_onehot_y=True needs a one-channel label map, got a %d-channel target" % tc)
        if c > 1 and not self.to_onehot_y and tc == 1:
            raise ValueError("a one-channel label map needs to_onehot_y=True (input has %d channels)" % c)

    def _class_weight(self, c: int, device):
        """the focal term's class factors as a CUDA tensor, or None"""
        return None

    def forward(self, input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        self._check_shapes(input, target)
        c = input.shape[1]
        out, tgt = _prepare(self._name, input, target)
        tgt, kind = self._target_kind(c, tgt)
        weight = self._class_weight(c, out.device)
        desc = _lib.dice_ce_desc(target_kind=kind, class_weight=weight, **self._opts)
        desc._class_weight = weight                          # the descriptor holds its address until the backward
        # fp64 scratch: the per-block partial sums, their totals and the backward coefficients
        scratch_len = _lib.dice_ce_scratch_bytes(desc, out.shape[0], c, out[0, 0].numel()) // 8
        with torch.cuda.device(out.device):
            return _DiceFunction.apply(out, tgt.contiguous(), desc, _lib.dice_ce_fwd, _lib.dice_ce_bwd, scratch_len)


def _act_opts(name, sigmoid, softmax, other_act):
    if other_act is not None:
        raise NotImplementedError("fused %s: other_act is not implemented" % name)
    if sigmoid and softmax:
        raise ValueError("Incompatible values: more than 1 of [sigmoid=True, softmax=True] are True.")
    return "softmax" if softmax else ("sigmoid" if sigmoid else None)


def _check_reduction(name, reduction):
    if reduction not in ("mean", "sum"):
        raise ValueError("fused %s: reduction=%r (only 'mean' / 'sum')" % (name, reduction))


def _focal_alpha(alpha, use_softmax, include_background):
    """MONAI's FocalLoss ignores alpha in the softmax form without the background channel (and warns)"""
    if alpha is not None and use_softmax and not include_background:
        warnings.warn("`include_background=False`, `alpha` ignored when using softmax.")
        return None
    return None if alpha is None else float(alpha)


class DiceCELoss(_FusedCriterion):
    """monai.losses.DiceCELoss: ``lambda_dice * Dice(act(input), target) + lambda_ce * CE(input, target)``.

    Dice is ``DiceLoss``'s formula on softmax, sigmoid or identity probabilities (``include_background=False`` drops channel 0
    after the activation); CE is computed on the raw logits: cross-entropy over the channels for C > 1 (a ``[N,1,...]`` label
    map, or a ``[N,C,...]`` class-probability target), ``BCEWithLogits`` for C == 1.  Label maps are read as stored in uint8
    or int64 (other dtypes through ``.long()``); a label outside ``[0, C)`` counts as an all-zero target row.  One-hot targets
    are uint8 (bool is taken as uint8) or fp32.  With C == 1, ``softmax`` and ``to_onehot_y`` are ignored, as in MONAI.
    Class weights and label smoothing are not implemented and raise.
    """

    _name = "DiceCELoss"

    def __init__(self, include_background=True, to_onehot_y=False, sigmoid=False, softmax=False, other_act=None,
                 squared_pred=False, jaccard=False, reduction="mean", smooth_nr=1e-5, smooth_dr=1e-5, batch=False,
                 weight=None, lambda_dice=1.0, lambda_ce=1.0, label_smoothing=0.0, ce_weight=None):
        super().__init__()
        if other_act is not None or weight is not None or ce_weight is not None or float(label_smoothing) != 0.0:
            raise NotImplementedError("fused DiceCELoss: other_act / weight / ce_weight / label_smoothing are not implemented")
        if sigmoid and softmax:
            raise ValueError("Incompatible values: more than 1 of [sigmoid=True, softmax=True] are True.")
        if reduction not in ("mean", "sum"):
            raise ValueError("fused DiceCELoss: reduction=%r (only 'mean' / 'sum')" % (reduction,))
        if lambda_dice < 0.0:
            raise ValueError("lambda_dice should be no less than 0.0.")
        if lambda_ce < 0.0:
            raise ValueError("lambda_ce should be no less than 0.0.")
        self.to_onehot_y = bool(to_onehot_y)
        self._opts = dict(act="softmax" if softmax else ("sigmoid" if sigmoid else None), include_background=include_background,
                          squared_pred=squared_pred, jaccard=jaccard, batch=batch, reduction=reduction, smooth_nr=smooth_nr,
                          smooth_dr=smooth_dr, lambda_dice=lambda_dice, lambda_ce=lambda_ce)


class TverskyLoss(_FusedCriterion):
    """monai.losses.TverskyLoss: per (n, c) (per c with ``batch``) on p = act(input),
    ``1 - (I + smooth_nr) / (I + alpha (P - I) + beta (T - I) + smooth_dr)`` with I = sum p t, P = sum p, T = sum t; the mean or
    sum over the terms.  Targets, activations and ``include_background`` as in ``DiceCELoss``."""

    _name = "TverskyLoss"

    def __init__(self, include_background=True, to_onehot_y=False, sigmoid=False, softmax=False, other_act=None, alpha=0.5,
                 beta=0.5, reduction="mean", smooth_nr=1e-5, smooth_dr=1e-5, batch=False):
        super().__init__()
        act = _act_opts(self._name, sigmoid, softmax, other_act)
        _check_reduction(self._name, reduction)
        self.to_onehot_y = bool(to_onehot_y)
        self._opts = dict(act=act, include_background=include_background, batch=batch, reduction=reduction, smooth_nr=smooth_nr,
                          smooth_dr=smooth_dr, lambda_dice=1.0, lambda_ce=0.0, overlap="tversky", tversky_alpha=alpha,
                          tversky_beta=beta)


class GeneralizedDiceLoss(_FusedCriterion):
    """monai.losses.GeneralizedDiceLoss: per sample (once with ``batch``)
    ``1 - (2 sum_c w_c I_c + smooth_nr) / (sum_c w_c (P_c + T_c) + smooth_dr)``, w_c = 1 / T_c^2 (``w_type="square"``), 1 / T_c
    (``"simple"``) or 1 (``"uniform"``); an infinite weight (an absent class) becomes the largest finite weight of the sample (of
    the batch, with ``batch``).  The weights carry no gradient.  Targets, activations and ``include_background`` as in
    ``DiceCELoss``."""

    _name = "GeneralizedDiceLoss"

    def __init__(self, include_background=True, to_onehot_y=False, sigmoid=False, softmax=False, other_act=None, w_type="square",
                 reduction="mean", smooth_nr=1e-5, smooth_dr=1e-5, batch=False):
        super().__init__()
        act = _act_opts(self._name, sigmoid, softmax, other_act)
        _check_reduction(self._name, reduction)
        w_type = str(w_type).lower()
        if w_type not in _lib.GDICE_WEIGHTS:
            raise ValueError("w_type=%r: one of %s" % (w_type, ", ".join(_lib.GDICE_WEIGHTS)))
        self.to_onehot_y = bool(to_onehot_y)
        self._opts = dict(act=act, include_background=include_background, batch=batch, reduction=reduction, smooth_nr=smooth_nr,
                          smooth_dr=smooth_dr, lambda_dice=1.0, lambda_ce=0.0, overlap="generalized_dice", w_type=w_type)


class FocalLoss(_FusedCriterion):
    """monai.losses.FocalLoss on the channels ``include_background`` keeps (the background is dropped before the activation).

    Sigmoid form (``use_softmax=False``), per element: ``(x - x t - logsigmoid(x)) exp(gamma logsigmoid(-x (2t - 1)))``, times
    ``t alpha + (1 - t)(1 - alpha)`` with ``alpha``.  Softmax form: ``-(1 - exp(ls))^gamma ls t`` with ls the log-softmax over
    the kept channels, times ``1 - alpha`` on the first kept channel and ``alpha`` on the others (``alpha`` is ignored without
    the background, as in MONAI).  ``weight``: a scalar or one factor >= 0 per kept channel (ignored with one kept channel).
    ``"mean"`` divides the total by N * C' * S; ``"sum"``, as MONAI, sums the per-(n, c) means over the voxels.
    """

    _name = "FocalLoss"

    def __init__(self, include_background=True, to_onehot_y=False, gamma=2.0, alpha=None, weight=None, reduction="mean",
                 use_softmax=False):
        super().__init__()
        _check_reduction(self._name, reduction)
        if float(gamma) < 0.0:
            raise ValueError("gamma=%r: the focal exponent should be no less than 0" % (gamma,))
        self.to_onehot_y = bool(to_onehot_y)
        self._weight = _check_weight(weight)
        self._weights = {}
        self._opts = dict(act=None, include_background=include_background, reduction=reduction, lambda_dice=0.0, lambda_ce=1.0,
                          voxel_term="focal", focal_softmax=use_softmax, focal_gamma=gamma,
                          focal_alpha=_focal_alpha(alpha, use_softmax, include_background))

    def _class_weight(self, c, device):
        kept = c - 1 if (not self._opts["include_background"] and c > 1) else c
        if self._weight is None or kept == 1:
            return None
        key = (str(device), kept)
        if key not in self._weights:                         # built once per device: a graphed step replays the same buffer
            w = self._weight
            if w.numel() == 1:
                w = w.reshape(1).expand(kept)
            if w.numel() != kept:
                raise ValueError("the length of the `weight` sequence should be the same as the number of classes "
                                 "(%d weights, %d classes)" % (w.numel(), kept))
            self._weights[key] = w.to(device=device, dtype=torch.float32).contiguous()
        return self._weights[key]


def _check_weight(weight):
    if weight is None:
        return None
    w = torch.as_tensor(weight, dtype=torch.float64).detach().cpu().reshape(-1)
    if bool((w < 0).any()):
        raise ValueError("the value/values of the `weight` should be no less than 0.")
    return w


class DiceFocalLoss(_FusedCriterion):
    """monai.losses.DiceFocalLoss: ``lambda_dice * DiceLoss(...) + lambda_focal * FocalLoss(..., use_softmax=softmax)`` on one
    target (one-hot conversion happens once).  Under ``softmax=True, include_background=False`` the two terms take different
    softmaxes: the Dice over all C channels (channel 0 dropped afterwards), the focal term over channels 1..C-1.  Class weights
    raise: the Dice side has none in this package."""

    _name = "DiceFocalLoss"

    def __init__(self, include_background=True, to_onehot_y=False, sigmoid=False, softmax=False, other_act=None,
                 squared_pred=False, jaccard=False, reduction="mean", smooth_nr=1e-5, smooth_dr=1e-5, batch=False, gamma=2.0,
                 weight=None, lambda_dice=1.0, lambda_focal=1.0, alpha=None):
        super().__init__()
        if weight is not None:
            raise NotImplementedError("fused DiceFocalLoss: weight is not implemented")
        act = _act_opts(self._name, sigmoid, softmax, other_act)
        _check_reduction(self._name, reduction)
        if lambda_dice < 0.0:
            raise ValueError("lambda_dice should be no less than 0.0.")
        if lambda_focal < 0.0:
            raise ValueError("lambda_focal should be no less than 0.0.")
        if float(gamma) < 0.0:
            raise ValueError("gamma=%r: the focal exponent should be no less than 0" % (gamma,))
        self.to_onehot_y = bool(to_onehot_y)
        self._opts = dict(act=act, include_background=include_background, squared_pred=squared_pred, jaccard=jaccard, batch=batch,
                          reduction=reduction, smooth_nr=smooth_nr, smooth_dr=smooth_dr, lambda_dice=lambda_dice,
                          lambda_ce=lambda_focal, voxel_term="focal", focal_softmax=softmax, focal_gamma=gamma,
                          focal_alpha=_focal_alpha(alpha, softmax, include_background))


class HausdorffDTLoss(_FusedCriterion):
    """monai.losses.HausdorffDTLoss (Karimi & Salcudean 2019), on 3-D ``[N, C, D, H, W]`` inputs of at most 256 voxels per axis.

    p = act(input) (sigmoid, softmax over all C channels, or identity); ``include_background=False`` then drops channel 0.  For
    every kept (n, c) the prediction mask p > 0.5 and the target mask t > 0.5 each get the distance field edt(mask) + edt(~mask)
    (Euclidean distance in voxels to the nearest voxel of the other value, as scipy's ``distance_transform_edt`` rounded to
    fp32; 0 for an empty or full mask), computed on the device and carrying no gradient.  ``f_nc = mean over the voxels (and n
    with ``batch``) of (p - t)^2 (pdt^alpha + tdt^alpha)``; the loss is the mean or sum of the f terms.  Targets, ``to_onehot_y``
    and the C == 1 rules as in ``DiceCELoss``; a label outside ``[0, C)`` is an all-zero target row.  ``other_act``, 2-D inputs,
    larger extents and ``alpha <= 0`` raise ``NotImplementedError``; ``reduction="none"`` raises ``ValueError``.
    """

    _name = "HausdorffDTLoss"

    def __init__(self, alpha=2.0, include_background=False, to_onehot_y=False, sigmoid=False, softmax=False, other_act=None,
                 reduction="mean", batch=False):
        super().__init__()
        if other_act is not None:
            raise NotImplementedError("fused %s: other_act is not implemented" % self._name)
        if not float(alpha) > 0.0:
            raise NotImplementedError("fused %s: alpha=%r (only alpha > 0)" % (self._name, alpha))
        act = _act_opts(self._name, sigmoid, softmax, other_act)
        _check_reduction(self._name, reduction)
        self.alpha = float(alpha)
        self.to_onehot_y = bool(to_onehot_y)
        self._opts = dict(act=act, include_background=include_background, batch=batch, reduction=reduction, lambda_dice=0.0,
                          lambda_ce=1.0, voxel_term="hausdorff_dt")

    def _check_extent(self, input: torch.Tensor) -> None:
        if input.dim() != 5:
            raise NotImplementedError("fused %s: only 3-D [N, C, D, H, W] inputs, got shape %s" % (self._name, tuple(input.shape)))
        if max(input.shape[2:]) > _SURFACE_MAX_EXTENT:
            raise NotImplementedError("fused %s: spatial extent %s; at most %d voxels per axis"
                                      % (self._name, tuple(input.shape[2:]), _SURFACE_MAX_EXTENT))

    def forward(self, input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        self._check_extent(input)
        self._check_shapes(input, target)
        n, c, d, h, w = input.shape
        out, tgt = _prepare(self._name, input, target)
        tgt, kind = self._target_kind(c, tgt)
        tgt = tgt.contiguous()
        kept = c - 1 if (not self._opts["include_background"] and c > 1) else c
        desc = _lib.dice_ce_desc(target_kind=kind, **self._opts)
        with torch.cuda.device(out.device):
            # the distance weights are constants of the loss: computed here, outside autograd, and held by the descriptor until
            # the backward has read them
            field_scratch = torch.empty(_lib.hausdorff_dt_scratch_bytes(desc, n, c, d, h, w), dtype=torch.uint8, device=out.device)
            weight = torch.empty((n, kept, d, h, w), dtype=torch.float32, device=out.device)
            _lib.hausdorff_dt_weight(desc, out, tgt, self.alpha, field_scratch, weight)
            desc.hdt_weight = weight.data_ptr()
            desc._hdt_weight = weight
            scratch_len = _lib.dice_ce_scratch_bytes(desc, n, c, d * h * w) // 8
            return _DiceFunction.apply(out, tgt, desc, _lib.dice_ce_fwd, _lib.dice_ce_bwd, scratch_len)


class LogHausdorffDTLoss(HausdorffDTLoss):
    """monai.losses.LogHausdorffDTLoss: ``log(HausdorffDTLoss + 1)``, same arguments."""

    _name = "LogHausdorffDTLoss"

    def forward(self, input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        return torch.log(super().forward(input, target) + 1)
