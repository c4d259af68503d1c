"""Dice, IoU and confusion-matrix metrics on the device against the numpy restatement of MONAI (tests/overlap_metrics_oracle.py):
the (P, G, I) counts equal the oracle's exactly, every per-pair Dice and IoU and the confusion matrix bit for bit, the confusion
metrics within 1 fp32 ulp and the reductions within 1e-6; at the launch geometries users run, bit-identical run to run, and
replayable from a CUDA graph."""
import zlib

import numpy as np
import pytest
import torch

import overlap_metrics_oracle as orc

pytestmark = pytest.mark.gpu

REDUCTIONS = ["none", "mean", "sum", "mean_batch", "sum_batch", "mean_channel", "sum_channel"]
# prediction forms: (DiceHelper flags, how y_pred is made)
PRED_FORMS = {
    "onehot_bool": dict(softmax=False), "onehot_u8": dict(softmax=False), "onehot_f32": dict(softmax=False),
    "label_u8": dict(softmax=False, label=True), "label_i64": dict(softmax=False, label=True),
    "sigmoid": dict(sigmoid=True, activate=True), "threshold": dict(sigmoid=True), "argmax": dict(softmax=True),
}
TARGET_FORMS = ["onehot_bool", "onehot_u8", "onehot_f32", "label_u8", "label_i64"]
_DT = {"bool": torch.bool, "u8": torch.uint8, "f32": torch.float32, "i64": torch.int64}


@pytest.fixture(scope="module")
def M(pkg):
    return pkg.metrics


def make_labels(rng, b, c, shape, outside=True):
    """label maps [b, 1, *shape] with blobs of each class over a background, and (outside) a few labels >= c"""
    lab = rng.integers(0, c, size=(b, 1) + shape)
    lab[rng.random(lab.shape) < 0.5] = 0
    if outside:
        lab[rng.random(lab.shape) < 0.02] = c + 3
    return lab


def make_input(rng, form, b, c, shape):
    """(numpy array the oracle reads, CUDA tensor) of one form"""
    kind, dt = form.split("_") if "_" in form else (form, "f32")
    if kind == "label":
        lab = make_labels(rng, b, c, shape)
        return lab, torch.from_numpy(lab).to(_DT[dt]).cuda()          # labels stay below 256: uint8 holds them
    if kind == "onehot":
        m = rng.random((b, c) + shape) < 0.3
        if dt == "f32":
            v = np.where(m, rng.choice([1.0, 0.25, -2.0], size=m.shape), 0.0).astype(np.float32)   # nonzero = class
            return v, torch.from_numpy(v).cuda()
        return m, torch.from_numpy(m).to(_DT[dt]).cuda()
    if kind == "threshold":
        v = rng.random((b, c) + shape, dtype=np.float32)
        v[..., 0] = 0.5                                                # exactly 0.5 is not above it
        return v, torch.from_numpy(v).cuda()
    v = rng.standard_normal(size=(b, c) + shape, dtype=np.float32)
    if kind == "sigmoid":
        v[..., 0] = 0.0
        v[..., 1] = np.float32(1e-8)                                   # sigmoid rounds to exactly 0.5
    else:
        np.round(v, out=v)                                             # many argmax ties
    return v, torch.from_numpy(v).cuda()


def oracle_counts(pred_np, form, y_np, c):
    flags = PRED_FORMS[form]
    if flags.get("activate"):
        # MONAI on a CUDA tensor: torch's device sigmoid, then > 0.5 (the CPU sigmoid crosses 0.5 at a larger x)
        pred_np = torch.sigmoid(torch.from_numpy(pred_np).cuda()).cpu().numpy()
    pm = orc.discretise(pred_np, c, sigmoid=flags.get("sigmoid", False), softmax=flags.get("softmax", False),
                        num_classes=c if flags.get("label") else None)
    return orc.counts(pm, orc.target_masks(y_np, c))


def helper(M, form, c, **kw):
    flags = {k: v for k, v in PRED_FORMS[form].items() if k != "label"}
    return M.DiceHelper(num_classes=c if PRED_FORMS[form].get("label") else None, **flags, **kw)


def ulp_equal(a, b, ulps=1):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    fin = np.isfinite(a) & np.isfinite(b)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    return bool(np.all(same | (fin & (np.abs(ia - ib) <= ulps))))


def exact(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def check_counts(M, pred, form, y, pred_np, y_np, c):
    P, G, I = (t.cpu().numpy() for t in helper(M, form, c, include_background=True).counts(pred, y))
    rP, rG, rI = oracle_counts(pred_np, form, y_np, c)
    assert np.array_equal(P, rP) and np.array_equal(G, rG) and np.array_equal(I, rI)
    return rP, rG, rI


@pytest.mark.parametrize("target", TARGET_FORMS)
@pytest.mark.parametrize("form", list(PRED_FORMS))
def test_forms_against_oracle(M, form, target):
    rng = np.random.default_rng(zlib.crc32((form + target).encode()))
    b, c, shape = 3, 4, (9, 10, 11)
    pred_np, pred = make_input(rng, form, b, c, shape)
    y_np, y = make_input(rng, target, b, c, shape)
    y_np[1] = 0                                                        # item 1: an all-zero target
    y[1] = 0
    rP, rG, rI = check_counts(M, pred, form, y, pred_np, y_np, c)
    for include_background in (True, False):
        P, G, I = orc.drop_background(rP, rG, rI, include_background)
        for ignore_empty in (True, False):
            ref = orc.dice(P, G, I, ignore_empty)
            for reduction in REDUCTIONS:
                f, nn = helper(M, form, c, include_background=include_background, ignore_empty=ignore_empty, reduction=reduction)(pred, y)
                rf, rnn = orc.reduce(ref, reduction)
                if reduction == "none":
                    assert exact(f.cpu().numpy(), rf)
                else:
                    np.testing.assert_allclose(f.cpu().numpy(), rf, rtol=1e-6, atol=0, equal_nan=True)
                np.testing.assert_array_equal(nn.cpu().numpy(), rnn)


@pytest.mark.parametrize("pdt", ["bool", "u8", "f32"])
@pytest.mark.parametrize("ydt", ["bool", "u8", "f32"])
def test_iou_and_confusion_against_oracle(M, pdt, ydt):
    rng = np.random.default_rng(7)
    b, c, shape = 2, 3, (7, 13, 6)
    pred_np, pred = make_input(rng, "onehot_" + pdt, b, c, shape)
    y_np, y = make_input(rng, "onehot_" + ydt, b, c, shape)
    y_np[0, 1] = 0
    y[0, 1] = 0
    S = int(np.prod(shape))
    rP, rG, rI = orc.counts(pred_np.reshape(b, c, -1) != 0, y_np.reshape(b, c, -1) != 0)
    for include_background in (True, False):
        P, G, I = orc.drop_background(rP, rG, rI, include_background)
        for ignore_empty in (True, False):
            assert exact(M.compute_iou(pred, y, include_background, ignore_empty).cpu().numpy(), orc.iou(P, G, I, ignore_empty))
            m = M.MeanIoU(include_background=include_background, ignore_empty=ignore_empty, reduction="mean_batch")
            m(pred, y)
            m(pred, y)
            f = m.aggregate().cpu().numpy()
            np.testing.assert_allclose(f, orc.reduce(np.concatenate([orc.iou(P, G, I, ignore_empty)] * 2), "mean_batch")[0], rtol=1e-6,
                                       equal_nan=True)
        cm = M.get_confusion_matrix(pred, y, include_background)
        rcm = orc.confusion_matrix(P, G, I, S)
        assert cm.dtype == torch.float32 and exact(cm.cpu().numpy(), rcm)
        for name in orc.CM_NAMES:
            assert ulp_equal(M.compute_confusion_matrix_metric(name, cm).cpu().numpy(), orc.cm_metric(name, rcm))
        for compute_sample in (False, True):
            for reduction in ("mean", "sum_batch"):
                cmm = M.ConfusionMatrixMetric(include_background, metric_name=list(orc.CM_NAMES), compute_sample=compute_sample,
                                              reduction=reduction, get_not_nans=True)
                cmm(pred, y)
                for name, (f, nn) in zip(orc.CM_NAMES, cmm.aggregate()):
                    if compute_sample:
                        rf, rnn = orc.reduce(orc.cm_metric(name, rcm), reduction)
                    else:
                        red, rnn = orc.reduce(rcm, reduction)
                        rf = orc.cm_metric(name, red)
                    f = f.cpu().numpy()
                    np.testing.assert_allclose(f, np.asarray(rf).reshape(f.shape), rtol=2e-6, atol=1e-7, equal_nan=True)
                    np.testing.assert_array_equal(nn.cpu().numpy(), rnn)


def test_dice_metric_cumulative_and_labels(M):
    rng = np.random.default_rng(11)
    c = 4
    batches = [(make_input(rng, "argmax", 2, c, (8, 8, 8)), make_input(rng, "label_u8", 2, c, (8, 8, 8))) for _ in range(3)]
    m = M.DiceMetric(include_background=False, reduction="mean_batch", return_with_label=True)
    refs = []
    for (pn, p), (yn, y) in batches:
        onehot = torch.nn.functional.one_hot(torch.argmax(p, 1), c).permute(0, 4, 1, 2, 3).to(torch.uint8)
        m(onehot, y)
        refs.append(orc.dice(*orc.drop_background(*oracle_counts(pn, "argmax", yn, c), False)))
    out = m.aggregate()
    rf, _ = orc.reduce(np.concatenate(refs), "mean_batch")
    assert sorted(out) == ["label_1", "label_2", "label_3"]
    assert [out[k] for k in sorted(out)] == [round(float(v), 4) for v in rf]
    m.return_with_label = False
    np.testing.assert_allclose(m.aggregate().cpu().numpy(), rf, rtol=1e-6)
    m.reset()
    assert m.get_buffer() is None


def _run_case(M, form, target, b, c, shape, seed):
    rng = np.random.default_rng(seed)
    pred_np, pred = make_input(rng, form, b, c, shape)
    y_np, y = make_input(rng, target, b, c, shape)
    rP, rG, rI = check_counts(M, pred, form, y, pred_np, y_np, c)
    d = helper(M, form, c, include_background=True, reduction="none", get_not_nans=False)(pred, y)
    assert exact(d.cpu().numpy(), orc.dice(rP, rG, rI))
    return pred, y


@pytest.mark.parametrize("name,form,target,b,c,shape", [
    ("brats", "sigmoid", "onehot_u8", 1, 3, (240, 240, 155)),
    ("c2", "argmax", "label_i64", 2, 3, (128, 128, 128)),
    ("c2_sigmoid", "sigmoid", "onehot_u8", 2, 3, (128, 128, 128)),
    ("classes104_argmax", "argmax", "label_u8", 2, 104, (128, 128, 128)),
    ("classes104_labels", "label_u8", "label_i64", 2, 104, (128, 128, 128)),
    ("non_pow2", "onehot_u8", "onehot_f32", 3, 5, (7, 11, 13)),
    ("large_bc", "label_i64", "onehot_u8", 512, 128, (4, 4, 5)),
    ("large_bc_argmax", "argmax", "label_u8", 300, 128, (3, 5, 7)),
])
def test_launch_geometries(M, name, form, target, b, c, shape):
    _run_case(M, form, target, b, c, shape, seed=len(name))


def test_edge_cases(M):
    # C = 1: one-hot and sigmoid against a one-channel target
    for form in ("onehot_u8", "sigmoid", "threshold"):
        _run_case(M, form, "onehot_u8", 2, 1, (5, 6, 7), seed=1)
    # argmax ties: every channel equal -> class 0 everywhere
    x = torch.zeros(2, 5, 4, 4, 4, device="cuda")
    y = torch.zeros(2, 1, 4, 4, 4, dtype=torch.uint8, device="cuda")
    P, G, I = M.DiceHelper(softmax=True, include_background=True).counts(x, y)
    assert P[:, 0].tolist() == [64, 64] and int(P[:, 1:].sum()) == 0 and I[:, 0].tolist() == [64, 64]
    # labels outside [0, C) in both operands count for no class
    lab = torch.tensor([0, 1, 2, 200, 255, 3, 1, 1], dtype=torch.uint8, device="cuda").view(1, 1, 2, 2, 2)
    gt = torch.tensor([-1, 1, 2, 2, 9, 3, 1, 2], dtype=torch.int64, device="cuda").view(1, 1, 2, 2, 2)
    P, G, I = M.DiceHelper(softmax=False, include_background=True, num_classes=4).counts(lab, gt)
    assert P.tolist() == [[1, 3, 1, 1]] and G.tolist() == [[0, 2, 3, 1]] and I.tolist() == [[0, 2, 1, 1]]
    # an all-empty batch: nan with ignore_empty, 1.0 without; the confusion matrix is all true negatives
    z = torch.zeros(2, 3, 6, 6, 6, dtype=torch.uint8, device="cuda")
    assert torch.isnan(M.compute_dice(z, z)).all()
    assert (M.compute_dice(z, z, ignore_empty=False) == 1).all()
    assert (M.compute_iou(z, z, ignore_empty=False) == 1).all()
    assert M.get_confusion_matrix(z, z)[..., 2].eq(216).all() and M.get_confusion_matrix(z, z)[..., [0, 1, 3]].eq(0).all()


def test_library_rejects_bad_arguments(pkg):
    lib = pkg.lib
    x = torch.zeros(1, 2, 2, 2, 2, device="cuda")
    counts = torch.empty(1, 2, 3, dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError, match="not supported"):
        lib.overlap_counts(x.to(torch.int64), "threshold", x, "onehot", 2, counts)
    with pytest.raises(RuntimeError, match="target kind 3"):
        lib.overlap_counts(x, "onehot", x, "argmax", 2, counts)
    with pytest.raises(RuntimeError, match="129 classes"):
        lib.overlap_counts(x, "onehot", x, "onehot", 129, counts)
    big = torch.zeros(65536, 1, 1, 1, 1, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="65536 items"):
        lib.overlap_counts(big, "onehot", big, "onehot", 1, torch.empty(65536, 1, 3, dtype=torch.int64, device="cuda"))


def test_bit_identical_run_to_run(M):
    pred, y = _run_case(M, "argmax", "label_u8", 2, 104, (64, 96, 80), seed=5)
    h = M.DiceHelper(softmax=True, include_background=True, reduction="none", get_not_nans=False)
    assert torch.equal(torch.stack(h.counts(pred, y)), torch.stack(h.counts(pred, y)))
    assert torch.equal(h(pred, y).view(torch.int32), h(pred, y).view(torch.int32))


def test_cuda_graph_capture_and_replay(M):
    rng = np.random.default_rng(9)
    pred_np, pred = make_input(rng, "sigmoid", 2, 3, (32, 40, 48))
    y_np, y = make_input(rng, "onehot_u8", 2, 3, (32, 40, 48))
    h = M.DiceHelper(sigmoid=True, activate=True, include_background=True, reduction="none", get_not_nans=False)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        h(pred, y)                                                     # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = h(pred, y)
    new_np, new = make_input(rng, "sigmoid", 2, 3, (32, 40, 48))
    pred.copy_(new)
    g.replay()
    torch.cuda.synchronize()
    assert exact(out.cpu().numpy(), orc.dice(*oracle_counts(new_np, "sigmoid", y_np, 3)))


def test_sigmoid_threshold_sweep_cuda(M):
    """x >= x* agrees with torch's CUDA sigmoid(x) > 0.5 on every fp32 from 2^17 ulps below x* to 2^17 ulps above where the CPU
    sigmoid crosses 0.5, both signs, and a log sweep; the kernel's count of the same values agrees"""
    x_star = np.float32(M.SIGMOID_ABOVE_HALF)
    near = np.arange(int(x_star.view(np.uint32)) - (1 << 17), 0x33C00001 + (1 << 17), dtype=np.int64).astype(np.uint32).view(np.float32)
    logs = np.concatenate([np.float32(10.0) ** np.linspace(-45, 38, 20001, dtype=np.float32), [0.0, np.inf, np.nan]]).astype(np.float32)
    x = np.concatenate([near, -near, logs, -logs]).astype(np.float32)
    xc = torch.from_numpy(x).cuda()
    ref = (torch.sigmoid(xc) > 0.5).cpu().numpy()
    assert np.array_equal(x >= x_star, ref)
    y = torch.ones(1, 1, 1, 1, x.size, dtype=torch.uint8, device="cuda")
    P, G, I = M.DiceHelper(sigmoid=True, activate=True).counts(xc.view(1, 1, 1, 1, -1), y)
    assert int(P) == int(ref.sum()) == int(I) and int(G) == x.size
