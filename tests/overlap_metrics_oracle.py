"""numpy restatement of MONAI's overlap metrics (monai/metrics/meandice.py, meaniou.py, confusion_matrix.py of MONAI 1.3+),
written from their per-channel loops and the rules metrics.py states: which form each DiceHelper flag selects, nonzero =
class for one-hot operands, a label outside [0, C) in no class, channel 0 dropped after counting, and MONAI's empty-mask rules.
Counts are exact int64; every score is formed in fp32 from them, in MONAI's order of operations."""
import numpy as np
import torch

CM_NAMES = {
    "tpr": ("sensitivity", "recall", "hit_rate", "true_positive_rate", "tpr"),
    "tnr": ("specificity", "selectivity", "true_negative_rate", "tnr"),
    "ppv": ("precision", "positive_predictive_value", "ppv"),
    "npv": ("negative_predictive_value", "npv"),
    "fnr": ("miss_rate", "false_negative_rate", "fnr"),
    "fpr": ("fall_out", "false_positive_rate", "fpr"),
    "fdr": ("false_discovery_rate", "fdr"),
    "for": ("false_omission_rate", "for"),
    "pt": ("prevalence_threshold", "pt"),
    "ts": ("threat_score", "critical_success_index", "ts", "csi"),
    "acc": ("accuracy", "acc"),
    "ba": ("balanced_accuracy", "ba"),
    "f1": ("f1_score", "f1"),
    "mcc": ("matthews_correlation_coefficient", "mcc"),
    "fm": ("fowlkes_mallows_index", "fm"),
    "bm": ("informedness", "bookmaker_informedness", "bm", "youden_index", "youden"),
    "mk": ("markedness", "deltap", "mk"),
}


def discretise(y_pred, n, *, sigmoid=False, softmax=False, activate=False, num_classes=None):
    """MONAI DiceHelper's choice of form: -> (mask [B, n, S] bool per class) of the prediction"""
    y_pred = np.asarray(y_pred)
    b = y_pred.shape[0]
    argmax, threshold = softmax, sigmoid
    if num_classes is not None and y_pred.shape[1] == 1 and n > 1:
        argmax = threshold = False
    flat = y_pred.reshape(b, y_pred.shape[1], -1)
    if argmax and n > 1:
        return one_hot_of_labels(np.argmax(flat, axis=1), n)
    if threshold:
        if activate:
            flat = torch.sigmoid(torch.from_numpy(np.ascontiguousarray(flat, np.float32))).numpy()
        return flat > 0.5
    if y_pred.shape[1] == 1 and n > 1:
        return one_hot_of_labels(flat[:, 0], n)
    return flat != 0


def one_hot_of_labels(lab, n):
    """[B, S] labels -> [B, n, S] bool; a label outside [0, n) is in no class"""
    lab = np.asarray(lab).astype(np.int64)
    return np.stack([lab == c for c in range(n)], axis=1)


def target_masks(y, n):
    """y [B, 1, ...] with n > 1 is a label map, else a one-hot [B, n, ...] (nonzero = class)"""
    y = np.asarray(y)
    flat = y.reshape(y.shape[0], y.shape[1], -1)
    if y.shape[1] == 1 and n > 1:
        return one_hot_of_labels(flat[:, 0], n)
    return flat != 0


def counts(pm, gm):
    """per-class masks [B, C, S] -> P, G, I int64 [B, C], one (item, class) pair at a time"""
    b, c = pm.shape[:2]
    P, G, I = (np.zeros((b, c), np.int64) for _ in range(3))
    for i in range(b):
        for k in range(c):
            P[i, k] = np.count_nonzero(pm[i, k])
            G[i, k] = np.count_nonzero(gm[i, k])
            I[i, k] = np.count_nonzero(pm[i, k] & gm[i, k])
    return P, G, I


def drop_background(P, G, I, include_background):
    if include_background or P.shape[1] == 1:
        return P, G, I
    return P[:, 1:], G[:, 1:], I[:, 1:]


def _score(num, den, G, P, ignore_empty):
    out = np.empty(G.shape, np.float32)
    for idx in np.ndindex(G.shape):
        if G[idx] > 0:
            out[idx] = np.float32(num[idx]) / np.float32(den[idx])
        elif ignore_empty:
            out[idx] = np.nan
        elif G[idx] + P[idx] == 0:
            out[idx] = 1.0
        else:
            out[idx] = 0.0
    return out


def dice(P, G, I, ignore_empty=True):
    """2I / (G + P) per pair; empty target: nan (ignore_empty), 1 if the prediction is empty too, else 0"""
    return _score(2 * I, G + P, G, P, ignore_empty)


def iou(P, G, I, ignore_empty=True):
    return _score(I, G + P - I, G, P, ignore_empty)


def confusion_matrix(P, G, I, S):
    """[B, C, 4] fp32 (tp, fp, tn, fn)"""
    return np.stack([I, P - I, S - P - G + I, G - I], axis=-1).astype(np.float32)


def metric_name(name):
    name = name.replace(" ", "_").lower()
    for short, aliases in CM_NAMES.items():
        if name in aliases:
            return short
    raise NotImplementedError(name)


def cm_metric(name, cm):
    """MONAI compute_confusion_matrix_metric in fp32, element by element"""
    m = metric_name(name)
    cm = np.asarray(cm, np.float32)
    out = np.empty(cm.shape[:-1], np.float32)
    one, two, nan = np.float32(1), np.float32(2), np.float32(np.nan)

    def ratio(a, b):
        return a / b if b > 0 else nan

    with np.errstate(all="ignore"):
        for idx in np.ndindex(out.shape):
            tp, fp, tn, fn = cm[idx]
            p, n = tp + fn, fp + tn
            den = None
            if m in ("pt", "ba", "bm"):
                tpr, tnr = ratio(tp, p), ratio(tn, n)
                if m == "pt":
                    num, den = np.sqrt(tpr * (one - tnr)) + tnr - one, tpr + tnr - one
                else:
                    out[idx] = (tpr + tnr) / two if m == "ba" else tpr + tnr - one
            elif m == "fm":
                out[idx] = np.sqrt(ratio(tp, tp + fp) * ratio(tp, p))
            elif m == "mk":
                out[idx] = ratio(tp, tp + fp) + ratio(tn, tn + fn) - one
            elif m == "mcc":
                num, den = tp * tn - fp * fn, np.sqrt((tp + fp) * (tp + fn) * (tn + fp) * (tn + fn))
            else:
                num, den = {"tpr": (tp, p), "tnr": (tn, n), "ppv": (tp, tp + fp), "npv": (tn, tn + fn), "fnr": (fn, p),
                            "fpr": (fp, n), "fdr": (fp, fp + tp), "for": (fn, fn + tn), "ts": (tp, tp + fn + fp),
                            "acc": (tp + tn, p + n), "f1": (tp * two, tp * two + fn + fp)}[m]
            if den is not None:
                out[idx] = num / den if den != 0 else nan
    return out


def reduce(f, reduction):
    """MONAI do_metric_reduction in numpy (nan left out; mean over channels, then batch)"""
    f = np.asarray(f, np.float32)
    nans = np.isnan(f)
    nn = (~nans).astype(np.float32)
    if reduction == "none":
        return f, nn
    g = np.where(nans, np.float32(0), f)
    if reduction == "mean":
        c = nn.sum(1)
        g = np.where(c > 0, g.sum(1) / np.maximum(c, 1), 0).astype(np.float32)
        b = (c > 0).sum(0).astype(np.float32)
        return np.where(b > 0, g.sum(0) / np.maximum(b, 1), 0).astype(np.float32), b
    if reduction == "sum":
        return g.sum((0, 1)), nn.sum((0, 1))
    if reduction == "mean_batch":
        b = nn.sum(0)
        return np.where(b > 0, g.sum(0) / np.maximum(b, 1), 0).astype(np.float32), b
    if reduction == "sum_batch":
        return g.sum(0), nn.sum(0)
    if reduction == "mean_channel":
        c = nn.sum(1)
        return np.where(c > 0, g.sum(1) / np.maximum(c, 1), 0).astype(np.float32), c
    if reduction == "sum_channel":
        return g.sum(1), nn.sum(1)
    raise ValueError(reduction)
