"""The GPU case table of FocalLoss, DiceFocalLoss, TverskyLoss and GeneralizedDiceLoss (tests/seg_loss_cases.py) reaches every
regime the new kernel paths have: both focal forms and the two-softmax voxel, every target kind, both kept-channel sets, batch,
sum, class weights, an absent generalized-Dice class, and blocks that loop over several tiles."""
import seg_loss_cases as S


def _keys():
    return {S.key(*case) for case in S.cases()}


def test_every_criterion_meets_every_class_count_and_target_form():
    seen = {(crit, c, form) for crit, _, c, form, _ in S.cases()}
    assert seen == {(crit, c, form) for crit in S.VARIANTS for c in S.CLASSES for form in S.FORMS}
    assert set(S.CLASSES) == {1, 3, 16, 104, 128}


def test_focal_regimes():
    keys = _keys()
    terms = {k[4] for k in keys}
    assert {"focal-sigmoid", "focal-softmax", "focal-two-softmax", "none"} <= terms
    # the two-softmax voxel on every target kind a label map or C-channel target launches with
    assert {k[2] for k in keys if k[4] == "focal-two-softmax"} == {"label_u8", "label_i64", "onehot_u8", "soft_f32"}
    # both focal forms with weights, without background, with sum
    for term in ("focal-sigmoid", "focal-softmax"):
        assert any(k[4] == term and k[8] == "weights" for k in keys), term
        assert any(k[4] == term and k[5] == "drop0" for k in keys), term
    assert any(k[4] == "focal-sigmoid" and k[7] == "sum" for k in keys)
    # one channel: the uint8 label map is launched as the one-hot target
    assert any(k[1] == "c1" and k[2] == "onehot_u8" and k[4] == "focal-sigmoid" for k in keys)


def test_overlap_regimes():
    keys = _keys()
    for crit in ("TverskyLoss", "GeneralizedDiceLoss", "DiceFocalLoss"):
        mine = [k for k in keys if k[0] == crit]
        assert {k[3] for k in mine} == {"none", "sigmoid", "softmax"}, crit
        assert {k[5] for k in mine} == {"all", "drop0"} and {k[6] for k in mine} == {"batch", "per-sample"}, crit
        assert {k[7] for k in mine} == {"mean", "sum"}, crit
    assert any(k[0] == "GeneralizedDiceLoss" and k[9] == "absent" and k[6] == "batch" for k in keys)
    assert any(k[0] == "GeneralizedDiceLoss" and k[9] == "absent" and k[6] == "per-sample" for k in keys)


def test_blocks_loop_over_several_tiles_at_many_classes():
    keys = _keys()
    assert {k[1] for k in keys if k[10] == "multi-tile"} >= {S.c_class(104)}
    assert any(k[10] == "one-tile" for k in keys)
