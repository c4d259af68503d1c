"""GPU cases of FocalLoss, DiceFocalLoss, TverskyLoss and GeneralizedDiceLoss on the Dice + cross-entropy kernels (csrc/dice_ce.cu,
csrc/dice.cu's finalize), and the regime each one puts the kernels in.

A case is (criterion, constructor kwargs, C, target form, spatial extent).  Its key names what the kernels do with it:
  (criterion, channel class, target kind as launched, Dice activation, per-voxel term, kept channels, batch, reduction,
   class weights, absent class, tiles per block)
  - per-voxel term: "none" (lambda_focal = 0 or no focal term), "focal-sigmoid", "focal-softmax", or "focal-two-softmax" (a
    softmax Dice over all C channels and a focal softmax over 1..C-1, one voxel needing both sums of exponentials);
  - kept channels: "all" or "drop0" (include_background = False with C > 1);
  - tiles per block from loss_prepost_cases.dice_ce_geometry (the launch code restated there).
tests/test_seg_loss_cases_host.py checks that the table reaches every regime; tests/test_gpu_seg_losses.py runs every case
against fp64 autograd of tests/seg_losses_oracle.py.
"""
from loss_prepost_cases import c_class, dice_ce_geometry

N = 2
CLASSES = (1, 3, 16, 104, 128)
FORMS = ("label_u8", "label_i64", "onehot_u8", "soft_f32")
WEIGHTS = "linspace"          # per-class factors 0.5 .. 2.0 over the kept channels, built by the runner

VARIANTS = {
    "FocalLoss": [dict(), dict(use_softmax=True), dict(use_softmax=True, include_background=False),
                  dict(include_background=False, alpha=0.25, reduction="sum"),
                  dict(use_softmax=True, gamma=0.0, alpha=0.3, weight=WEIGHTS), dict(gamma=0.5, weight=WEIGHTS, reduction="sum")],
    "DiceFocalLoss": [dict(softmax=True), dict(softmax=True, include_background=False), dict(sigmoid=True, batch=True, reduction="sum", alpha=0.25),
                      dict(softmax=True, include_background=False, batch=True, squared_pred=True, jaccard=True, lambda_dice=0.3,
                           lambda_focal=1.7, gamma=1.0),
                      dict(), dict(softmax=True, lambda_focal=0.0)],
    "TverskyLoss": [dict(softmax=True), dict(sigmoid=True, alpha=0.3, beta=0.7, batch=True),
                    dict(softmax=True, include_background=False, reduction="sum"), dict()],
    "GeneralizedDiceLoss": [dict(softmax=True), dict(sigmoid=True, w_type="simple", batch=True),
                            dict(softmax=True, include_background=False, w_type="uniform", reduction="sum"), dict()],
}


def spatial_of(c):
    """a partial last tile at few classes; several tiles per block at 104 and 128 classes"""
    return (32, 32, 32) if c >= 104 else (9, 11, 13)


def absent_class(crit, c, form):
    """generalized Dice cases on hard targets leave the last class out of sample 0: its square / simple weight is infinite"""
    return crit == "GeneralizedDiceLoss" and c > 1 and form != "soft_f32"


def cases():
    for crit, variants in VARIANTS.items():
        for c in CLASSES:
            for form in FORMS:
                for kw in variants:
                    yield crit, kw, c, form, spatial_of(c)


def key(crit, kw, c, form, spatial):
    act = "softmax" if kw.get("softmax") else ("sigmoid" if kw.get("sigmoid") else None)
    s = 1
    for v in spatial:
        s *= v
    g = dice_ce_geometry(N, c, s, form, act)
    drop0 = not kw.get("include_background", True) and c > 1
    if crit == "FocalLoss":
        smx = kw.get("use_softmax", False)
        term = "focal-softmax" if smx else "focal-sigmoid"
        act_l = "none"
    elif crit == "DiceFocalLoss" and kw.get("lambda_focal", 1.0) != 0.0:
        smx = bool(kw.get("softmax"))
        term = ("focal-two-softmax" if drop0 and g["act"] == "softmax" else "focal-softmax") if smx else "focal-sigmoid"
        act_l = g["act"] or "none"
    else:
        term, act_l = "none", g["act"] or "none"
    return (crit, c_class(c), g["kind"], act_l, term, "drop0" if drop0 else "all", "batch" if kw.get("batch") else "per-sample",
            kw.get("reduction", "mean"), "weights" if kw.get("weight") else "no-weights",
            "absent" if absent_class(crit, c, form) else "present", "multi-tile" if g["tiles_per_block"] > 1 else "one-tile")
