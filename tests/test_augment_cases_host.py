"""Every regime the training configurations put the augmentation and foreground-crop kernels in has a GPU case
(tests/augment_cases.py), every case still reaches the regime it is tagged with, and the restated launch rules still match the
constants in the sources.  The radix-select cases are checked against np.percentile through a numpy restatement of the three
passes.  Host only."""
import collections
import os
import re

import numpy as np
import pytest

import augment_cases as A

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "3dunetcnn_b200", "csrc")


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def test_launch_constants_match_the_sources():
    """a constant changed in augment.cu or foreground.cu without the restatement fails here"""
    for (fname, name), want in A.SOURCE_CONSTANTS.items():
        m = re.search(r"static constexpr int %s = ([^;]+);" % name, _source(fname))
        assert m, "%s not found in %s" % (name, fname)
        assert eval(m.group(1), {}) == want, (fname, name, m.group(1), want)          # noqa: S307 (an integer expression)
    aug = _source("augment.cu")
    assert "const long long cap = (132LL * 8 + N * C - 1) / (N * C);" in aug and A.AUG_INTENSITY_CAP == 132 * 8
    assert "((S + 3) / 4 + kAugThreads * 4 - 1) / (kAugThreads * 4)" in aug
    assert "if (C <= 4)\n    k_aug_resample<4>" in aug and "k_aug_resample<B200_AUG_MAX_CHANNELS>" in aug
    assert "#define B200_AUG_MAX_CHANNELS %d" % A.AUG_MAX_CHANNELS in _source("kernels.h")
    fg = _source("foreground.cu")
    assert "return pass == 0 ? 21 : pass == 1 ? 10 : 0;" in fg and "return pass == 2 ? 10 : 11;" in fg
    assert "(max_spatial + kFgThreads * kFgUnroll * 8 - 1) / (kFgThreads * kFgUnroll * 8)" in fg


def test_launch_rule_restatement():
    """spot values worked out by hand from augment.cu and foreground.cu"""
    # 2 x 4 x 128^3: 2097152 = 1024 x 2048, exactly at the cap; 192^3 = 7077888 = 3456 x 2048 -> 1024 blocks of 6912
    g = A.resample_geometry(128 ** 3)
    assert (g["nb"], g["per"], g["capped"], g["partial"], g["block_chain"], g["stats_chain"]) == (1024, 2048, False, False, 21, 12)
    g = A.resample_geometry(192 ** 3)
    assert (g["nb"], g["per"], g["capped"], g["partial"], g["block_chain"]) == (1024, 6912, True, False, 40)
    # 2146560 voxels: 1049 blocks wanted, 1024 of ceil(2146560 / 1024) = 2097, the last one 2146560 - 1023 x 2097 = 1329
    r = A.aug_block_ranges(2146560)
    assert len(r) == 1024 and r[0] == (0, 2097) and r[-1] == (1023 * 2097, 2146560) and r[-1][1] - r[-1][0] == 1329
    assert A.aug_block_ranges(1) == [(0, 1)] and A.aug_block_ranges(2049) == [(0, 1025), (1025, 2049)]
    assert [A.aug_cm(c) for c in (1, 4, 5, 16)] == [4, 4, 16, 16]
    assert A.stats_key(128 ** 3) == ("stats", "several") and A.stats_key(256 * 2048) == ("stats", "one")
    # intensity: 1 x 4 x 128^3 wants 512 chunks per plane, the cap is ceil(1056 / 4) = 264; 1100 planes: one block each
    assert A.intensity_launch(1, 4, 128 ** 3) == dict(chunks=264, capped=True, path="vec4")
    assert A.intensity_launch(100, 11, 4224) == dict(chunks=1, capped=True, path="vec4")
    assert A.intensity_launch(2, 3, 693, 4) == dict(chunks=1, capped=False, path="scalar")
    assert A.intensity_launch(2, 2, 7680, 4)["path"] == "unaligned" and A.intensity_launch(2, 2, 7680, 32)["path"] == "vec4"
    # foreground: 240 x 240 x 155 = 8928000 wants ceil(8928000 / 8192) = 1090 blocks; 4 planes: 264 each, 1 sample: 1056
    assert A.fg_blocks(8928000, 4) == (264, "capped") and A.fg_blocks(8928000, 1) == (1056, "capped")
    assert A.fg_blocks(9240, 1072) == (1, "one-per-row") and A.fg_blocks(8192, 1072) == (1, "uncapped")
    assert A.fg_blocks(1, 1) == (1, "uncapped")
    # 132 blocks over a 60-voxel sample: one voxel per block, 72 idle; 8928000 over 264: 33819 each, the last 34.2k short
    assert A.fg_idle([60], 132) and not A.fg_idle([8928000], 264) and A.fg_idle([9], 4) and not A.fg_idle([10], 4)
    # radix digits: bits 31..21, 20..10, 9..0; masks of the bits fixed before each pass
    assert [A.fg_mask(p) for p in range(3)] == [0, 0xFFE00000, 0xFFFFFC00]
    assert sum(A.FG_BITS) == 32 and max(1 << b for b in A.FG_BITS) == A.FG_BINS
    keys = A.fg_key(np.array([-np.inf, -1.0, -0.0, 0.0, 1.0, np.inf], dtype=np.float32))
    assert keys.tolist() == [0x007FFFFF, 0x407FFFFF, 0x80000000, 0x80000000, 0xBF800000, 0xFF800000]
    assert A.fg_value(keys).tolist() == [-np.inf, -1.0, 0.0, 0.0, 1.0, np.inf]
    assert A.divergence_pass(0xBF800000, 0xBF800800) == 1 and A.divergence_pass(0xBF800000, 0xBF800001) == 2
    assert A.divergence_pass(0x407FFFFF, 0x40800000) == 0 and A.divergence_pass(7, 7) == "none"


def test_percentile_index_is_the_package_one(pkg):
    for n in (1, 2, 3, 8, 1000, 40000, 8928000, 10485760, (1 << 24) + 3):
        for q in (0.0, 0.1, 0.25, 0.5, 0.9, 0.999, 1.0, 1.0 / 3.0):
            assert A.percentile_index(n, q) == pkg.augment.percentile_index(n, q), (n, q)


def test_case_reaches_its_regime():
    for c in A.RESAMPLE_CASES:
        assert c.key == c.tagged, c.id
        assert c.source == "batch" or len(c.samples) == c.n, c.id
        assert 1 <= c.c <= A.AUG_MAX_CHANNELS and c.n * c.c <= 65535, c.id
    for c in A.INTENSITY_CASES:
        assert c.key == c.tagged, c.id
    for c in A.FOREGROUND_CASES:
        assert c.keys == c.tagged, c.id
    for c in A.SELECT_CASES:
        assert A.select_pass(c.build(), c.percentile) == c.tagged, c.id


def _all_keys():
    have = collections.Counter()
    for c in A.RESAMPLE_CASES:
        have.update([c.key, A.stats_key(A.vol(c.out)), A.intensity_key(c.n, c.c, A.vol(c.out))])
    for c in A.INTENSITY_CASES:
        have.update([c.key] + ([A.stats_key(A.vol(c.dims))] if c.normalize else []))
    for c in A.FOREGROUND_CASES:
        have.update(k for k in c.keys if k is not None)
    for c in A.SELECT_CASES:
        have[("select", c.tagged)] += 1
    return have


def test_every_config_regime_has_a_case(pkg):
    keys = A.config_keys(pkg.augment)
    have = _all_keys()
    missing = {k: v for k, v in keys.items() if k not in have}
    assert not missing, "configuration regimes without a GPU case in tests/augment_cases.py: %r" % missing


def test_config_regimes_include_the_untested_geometry(pkg):
    """SPPIN's 192^3 output is above the resample block cap, and both datasets cap the foreground grids"""
    keys = A.config_keys(pkg.augment)
    assert keys[("resample", "samples", 4, "capped", "whole", "border")] == ["sppin"]
    assert keys[("resample", "samples", 4, "uncapped", "whole", "border")] == ["brats"]
    assert keys[("resample", "batch", 4, "uncapped", "whole", "border")] == ["batch-2x4x128"]
    assert keys[("fg-hist", "capped", "busy")] == ["brats", "sppin"] and ("fg-box", "capped", "several", "busy") in keys
    assert ("intensity", "vec4", "capped") in keys and ("stats", "several") in keys
    assert {k[1] for k in keys if k[0] == "select"} == {0, 1, 2, "none"}


def test_table_covers_the_edges():
    """the regimes no configuration reaches but the kernels accept"""
    have = _all_keys()
    assert {A.aug_cm(c.c) for c in A.RESAMPLE_CASES} == {4, 16}
    assert {c.c for c in A.RESAMPLE_CASES} >= {5, 8, 16}
    for cm in (4, 16):
        for pad in ("border", "zeros"):
            assert any(k[0] == "resample" and k[2] == cm and k[5] == pad for k in have), (cm, pad)
    assert {k[3] for k in have if k[0] == "resample"} == {"capped", "uncapped"}
    assert {k[4] for k in have if k[0] == "resample"} == {"partial", "whole"}
    assert ("resample", "batch", 4, "capped", "partial", "zeros") in have
    assert {(k[1], k[2]) for k in have if k[0] == "intensity"} >= {("vec4", "capped"), ("vec4", "uncapped"), ("scalar", "capped"),
                                                                  ("scalar", "uncapped"), ("unaligned", "uncapped")}
    assert any(c.offset and A.vol(c.dims) % 4 for c in A.INTENSITY_CASES)                      # S % 4 != 0, pointer off
    assert {("stats", "one"), ("stats", "several")} <= set(have)
    assert {k[1] for k in have if k[0] in ("fg-hist", "fg-box")} == {"uncapped", "capped", "one-per-row"}
    assert ("fg-hist", "one-per-row", "busy") in have and ("fg-box", "capped", "several", "idle") in have
    assert {c.tagged for c in A.SELECT_CASES} == {0, 1, 2, "none"}
    # the median of an even count: weight 0.5, where the interpolation switches to b - (b - a)(1 - t)
    assert any(A.percentile_index(c.n, c.percentile)[2] == np.float32(0.5) for c in A.SELECT_CASES)


def test_case_ids_are_unique():
    ids = collections.Counter(c.id for c in A.RESAMPLE_CASES + A.INTENSITY_CASES + A.FOREGROUND_CASES + A.SELECT_CASES)
    assert max(ids.values()) == 1, [i for i, k in ids.items() if k > 1]


def _same_value(a, b):
    """bit for bit, -0 as +0 and every NaN as one value"""
    a, b = np.float32(a), np.float32(b)
    if np.isnan(a) or np.isnan(b):
        return bool(np.isnan(a) and np.isnan(b))
    return (a + np.float32(0)).view(np.int32) == (b + np.float32(0)).view(np.int32)


@pytest.mark.parametrize("case", A.SELECT_CASES, ids=lambda c: c.id)
def test_select_restatement_reproduces_numpy(case):
    """the three passes restated in numpy give np.percentile bit for bit, keeping two histograms exactly after the pass the
    case diverges at"""
    x = case.build()
    assert x.dtype == np.float32 and x.size == case.n
    lo, hi, gamma = A.percentile_index(case.n, case.percentile)
    with np.errstate(invalid="ignore"):
        ref = np.percentile(x, case.percentile * 100)
    assert ref.dtype == np.float32
    thr, two_at = A.radix_select(x, lo, hi, gamma)
    assert _same_value(thr, ref), (case.id, thr, ref)
    d = case.tagged
    assert two_at == ([] if d == "none" else list(range(d + 1, 3))), (case.id, two_at)


def test_select_cases_are_sharp():
    """the weight-0.5 case tells numpy's b - (b - a)(1 - t) from a + (b - a) t, and the diverging cases interpolate between two
    different values with a non-zero weight"""
    sharp = []
    for c in A.SELECT_CASES:
        lo, hi, gamma = A.percentile_index(c.n, c.percentile)
        s = np.sort(c.build()[~np.isnan(c.build())])
        if gamma == np.float32(0.5):
            a, b = s[lo], s[hi]
            if np.float32(a + (b - a) * gamma) != A.lerp32(a, b, gamma):
                sharp.append(c.id)
        if c.tagged in (0, 1, 2) and c.fill != "nan" and not np.isinf(s[lo]):
            assert s[lo] != s[hi] and 0 < gamma < 1, c.id
    assert sharp == ["median-even"]


def test_too_many_planes_are_refused_without_a_launch(pkg):
    """k_fg_hist puts the n * c planes on gridDim.y (at most 65535): a larger batch is refused by the host-side size query, and
    launch_foreground_box returns E_UNSUPPORTED before it touches its (here bogus) pointers"""
    lib = pkg.lib.load_library()
    assert lib.b200unet_foreground_scratch_bytes(4095, 16) > 0 and lib.b200unet_foreground_scratch_bytes(65535, 1) > 0
    assert lib.b200unet_foreground_scratch_bytes(4096, 16) == 0 and lib.b200unet_foreground_scratch_bytes(4097, 16) == 0
    msg = lib.b200unet_last_error().decode()
    assert "n=4097" in msg and "c=16" in msg and "65535" in msg, msg
    bogus = 256
    st = lib.b200unet_foreground_box(bogus, 4097, 16, 1000, 1, bogus, bogus, 1, 1, bogus, 8, 8, 8, bogus, bogus, bogus, bogus, bogus,
                                     None)
    assert st == -2 and "n=4097" in lib.b200unet_last_error().decode()
