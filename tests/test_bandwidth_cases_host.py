"""Every regime the plans put the bandwidth-bound kernels in has a GPU case (tests/bandwidth_cases.py), and every case still
reaches the regime it is tagged with.  Host only: the launch rules are restated in Python."""
import collections

import pytest

import bandwidth_cases as B


def test_launch_rule_restatement():
    """spot values of the restated launch code, worked out by hand from elementwise.cu"""
    assert [B.ew_threads_for(c // 8) for c in (8, 24, 48, 96, 320, 384, 768, 1024)] == [256, 192, 192, 192, 160, 192, 192, 256]
    assert B.head_bwd_threads(48) == 288 and B.head_bwd_threads(24) == 288 and B.head_bwd_threads(32) == 256
    # GroupNorm at N = 2: 528 blocks; C = 32 (vper 64) needs S > 2 * 528 * 64 = 67,584 to run a second sweep
    assert B.gn_geometry(2, 32, (48, 48, 48))[:3] == (528, 256, True)
    assert B.gn_geometry(2, 32, (40, 40, 42))[2] is False
    assert B.gn_geometry(5, 32, (8, 8, 8))[0] == 4 and B.gn_geometry(5, 32, (48, 48, 48))[0] == 212   # 1056 / 5 rounds up
    assert B.gn_geometry(2, 768, (16, 16, 16))[2] and not B.gn_geometry(2, 768, (8, 8, 16))[2]
    assert B.act_bwd_geometry(2, 32, (16, 32, 34))[2] and not B.act_bwd_geometry(2, 32, (16, 32, 33))[2]
    assert B.upsample_bwd_kernel(False, (2, 4, 6)) == "blk"
    assert B.upsample_bwd_kernel(True, (2, 4, 6)) == B.upsample_bwd_kernel(False, (1, 4, 6)) == B.upsample_bwd_kernel(False, (3, 4, 6)) == "gather"
    assert B.bias_grad_geometry(2, 32, (128, 128, 128))[:3] == (592, 256, True)
    # SIMT head forward at the BraTS SegResNet size: 7,225,344 voxels over 2112 blocks of 256 threads, 13.4 sweeps
    assert B.head_fwd_geometry(1, 16, (224, 224, 144)) == (2112, 256, True, True)
    # head_dbias: 128 blocks per output; 220.5 sweeps of 32,768 voxels at 224 x 224 x 144, 64 exact ones at 128^3
    assert B.head_dbias_geometry(1, (224, 224, 144)) == (128, 256, True, True)
    assert B.head_dbias_geometry(2, (128, 128, 128)) == (128, 256, True, False)
    assert B.head_dbias_geometry(2, (24, 40, 32))[:3] == (120, 256, False)


@pytest.mark.parametrize("case", B.CASES, ids=lambda c: c.id)
def test_case_reaches_its_regime(case):
    assert B.regime_key(case.kernel, case.n, case.c, case.dims, case.split, case.view) == case.key


def test_every_plan_regime_has_a_case():
    have = {c.key for c in B.CASES}
    missing = {k: v[:2] for k, v in B.plan_keys().items() if k not in have}
    assert not missing, "plan regimes without a GPU case in tests/bandwidth_cases.py: %r" % missing


def test_plan_regimes_include_the_capped_grids():
    """the benchmark-size plans run every keyed kernel with a clamped grid, so the table must hold capped cases of each"""
    keys = B.plan_keys()
    capped = {k[0] for k in keys if k[2] == "capped"}
    assert capped >= {"gn", "act_bwd", "up_fwd", "up_add", "up_bwd_blk", "up_bwd_gather", "bias_grad", "head_bwd", "head_fwd",
                      "head_dbias"}
    assert ("up_fwd", "npow2", "capped", "tail", "bf16", "view") in keys          # C5: widths 48 .. 768
    assert any(k[0] == "gn" and k[1] == "wide" for k in keys)                     # C5 and BraTS: more than 256 channels


def test_case_ids_are_unique_and_each_kernel_has_both_precisions():
    ids = collections.Counter(c.id for c in B.CASES)
    assert max(ids.values()) == 1
    for kernel in {c.kernel for c in B.CASES} - {"head_dbias"}:     # k_head_dbias reads only the fp32 dlogits
        assert {c.split for c in B.CASES if c.kernel == kernel} == {False, True}, kernel
    assert {c.key[4] for c in B.CASES if c.kernel == "head_dbias"} == {"fp32"}


def test_gn_cases_hold_every_backward_variant_of_the_plans():
    """the regime key does not carry what k_gn_bwd adds and scales, so the variants the training plans hand it are checked here:
    each has a case in both precisions, and SegResNet's residual addend + Dropout3d scale also with a whole-buffer addend"""
    variants = B.plan_gn_bwd_variants()
    assert set(variants) == {"plain", "add1", "add1+scale"}
    assert any(name.startswith("brats-segresnet") for name in variants["add1+scale"])
    for v in variants:
        assert {c.split for c in B.GN_CASES if c.opt["bwd"] == v} == {False, True}, v
    assert {c.split for c in B.GN_CASES if c.opt["bwd"] == "add1+scale" and c.opt.get("whole")} == {False, True}
