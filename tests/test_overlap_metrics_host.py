"""Overlap metrics without a GPU: the numpy restatement of MONAI (tests/overlap_metrics_oracle.py) on hand-computed cases, every
empty-mask rule and every ConfusionMatrixMetric name and alias, argument validation, and the sigmoid threshold constant."""
import numpy as np
import pytest
import torch

import overlap_metrics_oracle as orc


@pytest.fixture(scope="module")
def M(pkg):
    return pkg.metrics


def test_oracle_counts_by_hand():
    # one item, 2 x 2 x 2 voxels, label maps over 3 classes; label 7 in the prediction and -1 in the target are in no class
    pred = np.array([0, 1, 1, 2, 2, 2, 7, 0]).reshape(1, 1, 2, 2, 2)
    gt = np.array([0, 1, 2, 2, 2, 0, 1, -1]).reshape(1, 1, 2, 2, 2)
    P, G, I = orc.counts(orc.discretise(pred, 3, num_classes=3), orc.target_masks(gt, 3))
    assert P.tolist() == [[2, 2, 3]]
    assert G.tolist() == [[2, 2, 3]]
    assert I.tolist() == [[1, 1, 2]]
    d = orc.dice(P, G, I)
    assert d.tolist() == [[np.float32(2 / 4), np.float32(2 / 4), np.float32(4 / 6)]]
    assert orc.iou(P, G, I).tolist() == [[np.float32(1 / 3), np.float32(1 / 3), np.float32(2 / 4)]]
    cm = orc.confusion_matrix(P, G, I, 8)
    assert cm[0, 2].tolist() == [2, 1, 4, 1]          # class 2: tp, fp, tn, fn
    P0, _, _ = orc.drop_background(P, G, I, False)
    assert P0.tolist() == [[2, 3]]


def test_oracle_forms():
    x = np.array([[-1.0, 3.0, 3.0, 0.0], [2.0, 3.0, -5.0, 0.0], [0.5, -1.0, 3.0, 0.0]], np.float32).reshape(1, 3, 1, 1, 4)
    am = orc.discretise(x, 3, softmax=True)           # argmax: ties go to the lowest channel
    assert np.argmax(am[0], axis=0).tolist() == [1, 0, 0, 0]
    th = orc.discretise(x, 3, sigmoid=True)           # x > 0.5 without the activation
    assert th[0].astype(int).tolist() == [[0, 1, 1, 0], [1, 1, 0, 0], [0, 0, 1, 0]]
    act = orc.discretise(x, 3, sigmoid=True, activate=True)
    assert act[0].astype(int).tolist() == [[0, 1, 1, 0], [1, 1, 0, 0], [1, 0, 1, 0]]
    one = orc.discretise(x, 3)                        # one-hot: nonzero
    assert one[0].astype(int).tolist() == [[1, 1, 1, 0], [1, 1, 1, 0], [1, 1, 1, 0]]


@pytest.mark.parametrize("ignore_empty", [True, False])
def test_oracle_empty_rules(ignore_empty):
    # pairs: target and prediction non-empty; target empty, prediction not; both empty
    P = np.array([[3, 2, 0]])
    G = np.array([[2, 0, 0]])
    I = np.array([[1, 0, 0]])
    d, j = orc.dice(P, G, I, ignore_empty), orc.iou(P, G, I, ignore_empty)
    assert d[0, 0] == np.float32(2 / 5) and j[0, 0] == np.float32(1 / 4)
    if ignore_empty:
        assert np.isnan(d[0, 1:]).all() and np.isnan(j[0, 1:]).all()
    else:
        assert d[0, 1:].tolist() == [0.0, 1.0] and j[0, 1:].tolist() == [0.0, 1.0]


def _cm_expect():
    tp, fp, tn, fn = 6.0, 2.0, 10.0, 4.0
    p, n = tp + fn, fp + tn
    tpr, tnr, ppv, npv = tp / p, tn / n, tp / (tp + fp), tn / (tn + fn)
    return (tp, fp, tn, fn), {
        "tpr": tpr, "tnr": tnr, "ppv": ppv, "npv": npv, "fnr": fn / p, "fpr": fp / n, "fdr": fp / (fp + tp), "for": fn / (fn + tn),
        "pt": (np.sqrt(tpr * (1 - tnr)) + tnr - 1) / (tpr + tnr - 1), "ts": tp / (tp + fn + fp), "acc": (tp + tn) / (p + n),
        "ba": (tpr + tnr) / 2, "f1": 2 * tp / (2 * tp + fn + fp),
        "mcc": (tp * tn - fp * fn) / np.sqrt((tp + fp) * (tp + fn) * (tn + fp) * (tn + fn)), "fm": np.sqrt(ppv * tpr),
        "bm": tpr + tnr - 1, "mk": ppv + npv - 1}


@pytest.mark.parametrize("alias", [a for aliases in orc.CM_NAMES.values() for a in aliases])
def test_confusion_metric_names_and_values(M, alias):
    cm, expect = _cm_expect()
    short = orc.metric_name(alias)
    assert M.check_confusion_matrix_metric_name(alias.upper().replace("_", " ")) == short
    ref = orc.cm_metric(alias, np.array([cm], np.float32))
    assert abs(float(ref[0]) - expect[short]) <= 1e-6 * max(1.0, abs(expect[short]))
    got = M.compute_confusion_matrix_metric(alias, torch.tensor([cm]))      # the torch formula runs on any device
    assert got.dtype == torch.float32
    assert abs(float(got[0]) - float(ref[0])) <= 1e-6 * max(1.0, abs(float(ref[0])))


@pytest.mark.parametrize("short", list(orc.CM_NAMES))
def test_confusion_metric_zero_denominators(M, short):
    cm = np.zeros((1, 4), np.float32)                 # nothing at all: every ratio has a zero denominator
    ref = orc.cm_metric(short, cm)
    got = M.compute_confusion_matrix_metric(short, torch.from_numpy(cm)).numpy()
    assert np.isnan(ref).all() and np.isnan(got).all()


def test_confusion_metric_name_errors(M):
    with pytest.raises(NotImplementedError):
        M.check_confusion_matrix_metric_name("dice")
    with pytest.raises(NotImplementedError):
        M.ConfusionMatrixMetric(metric_name=["f1", "nope"])
    with pytest.raises(ValueError, match="last dimension"):
        M.compute_confusion_matrix_metric("f1", torch.zeros(2, 3))


X_STAR_CPU = 0x33C00001        # where torch's CPU sigmoid crosses 0.5; the device's sigmoid crosses it 953833 fp32 values lower


def test_sigmoid_threshold_constant(M):
    x_star = np.float32(M.SIGMOID_ABOVE_HALF)
    assert x_star.view(np.uint32) == 0x33B17218
    assert X_STAR_CPU - 0x33B17218 == 953833
    cpu_star = np.uint32(X_STAR_CPU).view(np.float32)
    assert float(torch.sigmoid(torch.tensor(cpu_star))) > 0.5
    assert float(torch.sigmoid(torch.tensor(np.nextafter(cpu_star, np.float32(0))))) == 0.5
    assert float(torch.sigmoid(torch.tensor(np.float32(1e-30)))) == 0.5      # x > 0 is not the same test


def test_sigmoid_threshold_sweep_cpu(M):
    """every fp32 from 2^17 ulps below x* to 2^17 ulps above X_STAR_CPU (both signs), and a log sweep: x >= x* agrees with torch's CPU sigmoid(x) > 0.5 except on
    exactly the fp32 values in [x*, X_STAR_CPU), where only the device's sigmoid is above 0.5 (tests/test_gpu_overlap_metrics.py
    sweeps the same values against it)"""
    x_star = np.float32(M.SIGMOID_ABOVE_HALF)
    near = np.arange(int(x_star.view(np.uint32)) - (1 << 17), X_STAR_CPU + (1 << 17), dtype=np.int64).astype(np.uint32).view(np.float32)
    logs = np.concatenate([np.float32(10.0) ** np.linspace(-45, 38, 20001, dtype=np.float32), [0.0, np.inf, np.nan]]).astype(np.float32)
    x = np.concatenate([near, -near, logs, -logs]).astype(np.float32)
    ref = (torch.sigmoid(torch.from_numpy(x)) > 0.5).numpy()
    window = (x >= x_star) & (x < np.uint32(X_STAR_CPU).view(np.float32))
    assert np.array_equal((x >= x_star) & ~window, ref)
    assert np.count_nonzero(window[:near.size]) == 953833


def test_argument_validation(M):
    cpu = torch.zeros(1, 2, 4, 4, 4, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="CUDA"):
        M.compute_dice(cpu, cpu)
    with pytest.raises(RuntimeError, match="CUDA"):
        M.compute_iou(cpu, cpu)
    with pytest.raises(RuntimeError, match="CUDA"):
        M.get_confusion_matrix(cpu, cpu)
    with pytest.raises(ValueError, match="at least 3"):
        M.compute_dice(torch.zeros(2, 3), torch.zeros(2, 3))
    with pytest.raises(NotImplementedError, match="3-D"):
        M.compute_dice(torch.zeros(1, 2, 4, 4), torch.zeros(1, 2, 4, 4))
    with pytest.raises(ValueError, match="same shapes"):
        M.compute_iou(cpu, cpu[:, :1])
    with pytest.raises(ValueError, match="same batch and spatial"):
        M.compute_dice(cpu, cpu[..., :2])
    with pytest.raises(TypeError, match="dtype torch.int32"):
        M.compute_dice(cpu.int(), cpu)
    with pytest.raises(TypeError, match="label"):
        M.compute_dice(torch.zeros(1, 1, 4, 4, 4), cpu[:, :1], num_classes=3)       # fp32 label map
    with pytest.raises(TypeError, match="argmax"):
        M.DiceHelper(softmax=True)(cpu, cpu)                                        # argmax takes fp32 logits
    with pytest.raises(ValueError, match="channels"):
        M.compute_dice(cpu, cpu[:, :1].expand(1, 3, 4, 4, 4), num_classes=2)
    with pytest.raises(ValueError, match="1..128"):
        M.compute_dice(cpu[:, :1], cpu[:, :1], num_classes=129)
    with pytest.raises(TypeError):
        M.DiceMetric()(cpu, cpu, spacing=1.0)


def test_helper_flag_defaults(M):
    h = M.DiceHelper()
    assert (h.include_background, h.softmax, h.sigmoid, h.get_not_nans, h.reduction) == (False, True, False, True, "mean_batch")
    h = M.DiceHelper(sigmoid=True)
    assert (h.include_background, h.softmax) == (True, False)
    m = M.DiceMetric()
    assert (m.include_background, m.reduction, m.get_not_nans, m.ignore_empty, m.num_classes) == (True, "mean", False, True, None)
    c = M.ConfusionMatrixMetric()
    assert c.metric_name == ("hit_rate",) and not c.compute_sample


def test_exports(pkg):
    for name in ("DiceMetric", "MeanIoU", "ConfusionMatrixMetric", "HausdorffDistanceMetric"):
        assert getattr(pkg, name) is getattr(pkg.metrics, name)


@pytest.mark.parametrize("reduction", ["none", "mean", "sum", "mean_batch", "sum_batch", "mean_channel", "sum_channel"])
def test_oracle_reduction_matches_do_metric_reduction(M, reduction):
    rng = np.random.default_rng(3)
    f = rng.random((4, 5)).astype(np.float32)
    f[rng.random((4, 5)) < 0.3] = np.nan
    f[2] = np.nan
    ref, ref_nn = orc.reduce(f, reduction)
    got, got_nn = M.do_metric_reduction(torch.from_numpy(f), reduction)
    np.testing.assert_allclose(got.numpy(), ref, rtol=1e-6, equal_nan=True)
    np.testing.assert_array_equal(got_nn.numpy(), ref_nn)
