"""Fused Dice and Dice + cross-entropy criteria -- the classes ``load_criterion`` finds first.

The reference resolves ``config["loss"]["name"]`` in ``unet3d.losses`` before ``torch.nn`` and ``monai.losses``
(/root/reference/unet3d/scripts/script_utils.py:64-73; the shipped module is an empty hook,
unet3d/losses/losses.py:1-3), so a class named ``DiceLoss`` placed here takes over
``{"name": "DiceLoss", "include_background": true, "sigmoid": true}``
(examples/brats2020/brats2020_config.json:112-116) with MONAI's kwarg names.  Forward and backward are the
hand-written kernels ``b200unet_dice_fwd`` / ``b200unet_dice_bwd``; targets stay uint8 in HBM.  ``DiceCELoss`` takes over
``{"name": "DiceCELoss", "softmax": true, "to_onehot_y": true}`` the same way, on ``b200unet_dice_ce_fwd`` / ``_bwd``: it reads
a one-channel label map (or a C-channel target) and adds cross-entropy to a softmax Dice.
"""
from __future__ import annotations

import torch
from torch import nn

from . import lib as _lib


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


class DiceCELoss(nn.Module):
    """monai.losses.DiceCELoss: ``lambda_dice * Dice(act(input), target) + lambda_ce * CE(input, target)``.

    Dice is ``DiceLoss``'s formula on softmax, sigmoid or identity probabilities (``include_background=False`` drops channel 0
    after the activation); CE is computed on the raw logits: cross-entropy over the channels for C > 1 (a ``[N,1,...]`` label
    map, or a ``[N,C,...]`` class-probability target), ``BCEWithLogits`` for C == 1.  Label maps are read as stored in uint8
    or int64 (other dtypes through ``.long()``); a label outside ``[0, C)`` counts as an all-zero target row.  One-hot targets
    are uint8 (bool is taken as uint8) or fp32.  With C == 1, ``softmax`` and ``to_onehot_y`` are ignored, as in MONAI.
    Class weights and label smoothing are not implemented and raise.
    """

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

    def forward(self, input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
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
        out, tgt = _prepare("DiceCELoss", input, target)
        tgt, kind = self._target_kind(c, tgt)
        desc = _lib.dice_ce_desc(target_kind=kind, **self._opts)
        # fp64 scratch: the per-block partial sums, their totals and the backward coefficients
        scratch_len = _lib.dice_ce_scratch_bytes(desc, out.shape[0], c, out[0, 0].numel()) // 8
        with torch.cuda.device(out.device):
            return _DiceFunction.apply(out, tgt.contiguous(), desc, _lib.dice_ce_fwd, _lib.dice_ce_bwd, scratch_len)
