"""Every regime the configurations put the Dice, Dice + cross-entropy, tiling and z-score kernels in has a GPU case
(tests/loss_prepost_cases.py), and every case still reaches the regime it is tagged with.  Host only: the launch rules are
restated in Python."""
import collections

import pytest

import loss_prepost_cases as B


def test_launch_rule_restatement():
    """spot values of the restated launch code, worked out by hand from dice.cu, dice_ce.cu and prepost.cu"""
    # dice, C2: ceil(128^3 / 1024) = 2048 chunks capped at ceil(1056 / 6) = 176; 176 * 256 threads over 128^3 / 4 float4s
    # = 11.6 -> 12 sweeps of 4 terms
    assert B.dice_geometry(2, 3, 128 ** 3, "u8") == dict(chunks=176, capped=True, path="vec", sweeps=12, chain=48)
    # 104 / 128 outputs at N = 2: ceil(1056 / 208) = 6 and ceil(1056 / 256) = 5 blocks per (n, c); at 128^3 a thread adds
    # 128^3 / (6 * 256) = 1365.3 and 128^3 / (5 * 256) = 1638.4 terms
    assert B.dice_geometry(2, 104, 128 ** 3, "u8")["chunks"] == 6 and B.dice_geometry(2, 104, 128 ** 3, "u8")["chain"] == 4 * 342
    assert B.dice_geometry(2, 128, 128 ** 3, "u8")["chunks"] == 5 and B.dice_geometry(2, 128, 128 ** 3, "u8")["chain"] == 4 * 410
    # uncapped vector path: ceil(S / 1024) blocks of 256 threads hold S / 4 float4s, so one sweep; the scalar path needs four
    assert B.dice_geometry(1, 3, 32 ** 3, "u8")["sweeps"] == 1 and B.dice_geometry(1, 3, 32 ** 3, "f32")["sweeps"] == 4
    assert B.dice_geometry(2, 3, 105, "u8")["path"] == "scalar" and B.dice_geometry(2, 3, 32 ** 3, "u8", aligned=False)["path"] == "unaligned"
    # dice_ce, C = 3 label map: 8*128*3 + 4*3*129 + 512 + 512 = 5644 bytes -> 233472 / 6668 = 35 blocks per SM, clamped to 16;
    # 132 * 16 / 2 = 1056 blocks per sample over 16384 tiles: 16 tiles per block (15.5 on average)
    g = B.dice_ce_geometry(2, 3, 128 ** 3, "label_u8", "softmax")
    assert (g["smem"], g["grid_x"], g["tiles_per_block"], g["K"], g["idle"]) == (5644, 1056, 16, 42, 2)
    # C = 128 one-hot: 3072 + 2 * 4 * 128 * 129 + 1024 = 136192 bytes, one block per SM
    assert B.tile_smem(128, "onehot_u8") == 136192 and B.grid_x(1, 128, 128 ** 3, "onehot_u8") == 132
    assert B.grid_x(2, 104, 40 * 40 * 41, "label_u8") == 198            # 233472 / (3072 + 53664 + 1024 + 1024) = 3 per SM
    # test_gpu_dice_ce.py's largest shape: 240 tiles, 1056 blocks allowed -> one tile per block
    assert B.dice_ce_geometry(2, 3, 24 * 32 * 40, "label_u8", "softmax")["tiles_per_block"] == 1
    assert B.dice_ce_effective(1, "label_u8", "softmax") == ("onehot_u8", None)
    # tiling, C5: starts 0, 96, 128 per axis -> 27 tiles in 9 batches of 3; 3 * 128^3 / 256 = 24576 blocks, capped at 2112
    g = B.tiling_geometry((1, 1, 256, 256, 256), (128, 128, 128), 0.25, 3, 1)
    assert g["axes"] == [[0, 96, 128]] * 3 and (g["jobs"], g["batches"]) == (27, 9) and all(g["capped"].values())
    assert not g["spans"] and not g["partial"] and g["max_cover"] == 8
    assert B.grid_for(2112 * 256) == (2112, False) and B.grid_for(2112 * 256 + 1) == (2112, True)
    # 8 tiles per sample in batches of 5: the second batch holds tiles 5..9, of both samples
    g = B.tiling_geometry((2, 3, 20, 24, 28), (16, 16, 16), 0.25, 5, 2)
    assert g["spans"] and g["partial"] and not g["clamped"]
    assert B.tiling_geometry((1, 1, 12, 40, 12), (16, 16, 16), 0.25, 1, 3)["roi"] == (12, 16, 12)
    # z-score, BraTS: 4 groups -> 264 chunks (ceil(128^3 / 1024) = 2048 would be more); 32 sweeps at 128^3, 133 at 240^2 x 155
    assert B.zscore_geometry(4, 128 ** 3) == dict(chunks=264, capped=True, sweeps=32)
    assert B.zscore_geometry(4, 240 * 240 * 155)["sweeps"] == 133
    assert B.zscore_geometry(4, 20 * 24 * 28) == dict(chunks=14, capped=False, sweeps=4)


@pytest.mark.parametrize("case", B.CASES, ids=lambda c: c.id)
def test_case_reaches_its_regime(case):
    assert B.KEY_OF[case.kernel](*case.args) == case.key


def test_every_config_regime_has_a_case():
    have = {c.key for c in B.CASES}
    missing = {k: v[:2] for k, v in B.config_keys().items() if k not in have}
    assert not missing, "configuration regimes without a GPU case in tests/loss_prepost_cases.py: %r" % missing


def test_config_regimes_include_the_untested_geometry():
    """the benchmark-size configurations reach the capped Dice grid, several tiles per DiceCE block and the capped tiling and
    z-score grids, so the table must hold cases of each"""
    keys = B.config_keys()
    assert ("dice", "few", "capped", "multi-sweep", "vec", "u8") in keys                    # C2, C3, BraTS
    assert ("dice", "many", "capped", "multi-sweep", "vec", "u8") in keys                   # 104 outputs
    assert any(k[0] == "dice_ce" and k[5] == "multi-tile" for k in keys)
    assert ("tiles", "capped", "within", "full-last", "roi") in keys                         # C5
    assert ("zscore", "capped", "nonzero", "channel-wise") in keys                           # BraTS


def test_many_class_dice_runs_at_the_c2_size():
    """README's head table puts DiceLoss at 104 and 128 classes on 2 x 128^3: the table runs both shapes, so the longest
    per-thread chains (4 x 342 and 4 x 410 terms) are held to the bound model"""
    configs = {name: args for name, kernel, args in B.config_launches() if kernel == "dice"}
    assert configs["C2-104"] == (2, 104, 128 ** 3, "u8") and configs["C2-128"] == (2, 128, 128 ** 3, "u8")
    rows = {c.args[:4] for c in B.DICE_CASES if not c.opts}
    for n, c, S, t in (configs["C2-104"], configs["C2-128"]):
        assert (n, c, S, t) in rows
    chains = [B.dice_geometry(*c.args)["chain"] for c in B.DICE_CASES]
    assert max(chains) == 4 * 410 and 4 * 342 in chains


def test_table_covers_every_target_form_activation_and_edge():
    """beyond the configurations: both Dice target forms and the misaligned views; every DiceCE target form, activation, CE on
    and off, one and several tiles, partial tiles and idle threads; tile batches that span samples and end partial"""
    keys = {c.key for c in B.CASES}
    assert {k[5] for k in keys if k[0] == "dice"} == {"u8", "f32"}
    assert {k[4] for k in keys if k[0] == "dice"} == {"vec", "scalar", "unaligned"}
    assert {k[1] for k in keys if k[0] == "dice"} == {"c1", "few", "many"}
    dce = [k for k in keys if k[0] == "dice_ce"]
    assert {k[2] for k in dce} == set(B.TARGET_KINDS) and {k[3] for k in dce} == {"none", "sigmoid", "softmax"}
    for i, vals in ((1, {"c1", "few", "many"}), (4, {"ce", "no-ce"}), (5, {"one-tile", "multi-tile"}),
                    (6, {"partial-tile", "whole-tiles"}), (7, {"idle", "no-idle"})):
        assert {k[i] for k in dce} == vals
    assert ("tiles", "capped", "spans", "partial-last", "roi") in keys
    assert any(k[0] == "tiles" and k[4] == "clamped" for k in keys)
    assert {(k[2], k[3]) for k in keys if k[0] == "zscore"} == {("nonzero", "channel-wise"), ("all", "channel-wise"),
                                                               ("nonzero", "whole"), ("all", "whole")}
    assert {c.opt.get("misaligned") for c in B.DICE_CASES} == {None, "target", "logits"}


def test_case_ids_are_unique():
    ids = collections.Counter(c.id for c in B.CASES)
    assert max(ids.values()) == 1, [i for i, k in ids.items() if k > 1]
