"""Every regime the configurations put the 9..128-output tensor-core head in has a GPU case (tests/head_cases.py), and every
case still reaches the regime it is tagged with.  Host only: the launch rules are restated in Python."""
import collections

import head_cases as H


def test_launch_rule_restatement():
    """spot values of the restated launch code, worked out by hand from head.cu"""
    # C2: 2 x 128^3 = 4194304 voxels = 32768 tiles; 32768 = 124 x 264 + 32 and 248 x 132 + 32, so 32 forward CTAs walk 125
    # tiles and the other 232 walk 124; 32 backward slots hold 249 tiles and 100 hold 248
    g = H.head_geometry(104, 32, 2, (128, 128, 128))
    assert (g["tiles"], g["fwd_grid"], g["fwd_per_cta"], g["slots"], g["bwd_per_cta"]) == (32768, 264, 125, 132, 249)
    assert not g["fwd_even"] and not g["bwd_even"] and not g["partial"] and not g["straddle"] and g["path"] == "vec"
    assert g["tiles"] - (g["fwd_per_cta"] - 1) * g["fwd_grid"] == 32 and g["tiles"] - (g["bwd_per_cta"] - 1) * g["slots"] == 32
    # 104 outputs: NT 7, NP 112, NG 128, warpgroup 1 computes dw; 16 outputs: NT 1, NG 64, warpgroup 1 idle for dw
    assert (g["NT"], g["NP"], g["NG"], g["wg1_dw"]) == (7, 112, 128, True)
    g = H.head_geometry(16, 8, 1, (32, 32, 32))
    assert (g["NT"], g["NP"], g["NG"], g["wg1_dw"], g["ksteps"], g["kpad"]) == (1, 16, 64, False, 1, True)
    assert H.head_geometry(65, 64, 1, (4, 4, 8))["NT"] == 5 and not H.head_geometry(65, 64, 1, (4, 4, 8))["kpad"]
    # mc24 (1 x 32^3): 256 tiles, one per forward CTA; 256 = 132 + 124 over the backward slots, so two on 124 of them
    g = H.head_geometry(24, 8, 1, (32, 32, 32))
    assert (g["fwd_grid"], g["fwd_per_cta"], g["fwd_even"], g["slots"], g["bwd_per_cta"], g["bwd_even"]) == (256, 1, True, 132, 2, False)
    # 2 x 16^3: 64 tiles, 64 CTAs in both directions
    g = H.head_geometry(104, 8, 2, (16, 16, 16))
    assert (g["fwd_grid"], g["slots"], g["fwd_per_cta"], g["bwd_per_cta"]) == (64, 64, 1, 1)
    # the former kernel tests' 2 x 8 x 9 x 10: 1440 voxels = 11 tiles + 32, the 720-voxel samples meet inside tile 5
    g = H.head_geometry(9, 48, 2, (8, 9, 10))
    assert (g["tiles"], g["partial"], g["straddle"], g["path"]) == (12, True, True, "vec")
    # sweep shape A: S = 43993 (odd: scalar path), 87986 voxels = 687 tiles + 50; 688 = 2 x 264 + 160 and 5 x 132 + 28
    g = H.head_geometry(33, 24, *H.SHAPE_A)
    assert (g["S"], g["tiles"], g["fwd_per_cta"], g["bwd_per_cta"], g["path"]) == (43993, 688, 3, 6, "scalar")
    assert g["partial"] and g["straddle"] and not g["fwd_even"] and not g["bwd_even"]
    # sweep shape B: 528 tiles = 2 x 264 = 4 x 132
    g = H.head_geometry(48, 24, *H.SHAPE_B)
    assert (g["tiles"], g["fwd_per_cta"], g["fwd_even"], g["bwd_per_cta"], g["bwd_even"]) == (528, 2, True, 4, True)
    assert not g["partial"] and not g["straddle"]
    # a contiguous dlogits one float into its storage: S % 4 == 0 but the vector path is not taken
    assert H.head_geometry(104, 32, *H.SHAPE_B, aligned=False)["path"] == "unaligned"
    # shape D: S % 4 == 0 and the samples meet inside tiles
    g = H.head_geometry(40, 24, *H.SHAPE_D)
    assert (g["S"] % 4, g["straddle"], g["path"]) == (0, True, "vec")


def test_case_reaches_its_regime():
    """the hand-worked regime each row is tagged with is the one the restated launch code puts it in"""
    for case in H.CASES:
        g = case.geometry
        assert (case.fwd_key, case.bwd_key) == case.tagged_keys, case.id
        assert 9 <= case.n_out <= 128 and case.c % 8 == 0 and 8 <= case.c <= H.KMAXC
        assert case.ld is None or (case.ld % 8 == 0 and case.ld >= case.c + 8), case.id   # views start at channel 8
        assert case.offset == 0 or g["S"] % 4 == 0, case.id                                 # only then is there a vector path to leave


def test_every_config_regime_has_a_case():
    have = {c.fwd_key for c in H.CASES} | {c.bwd_key for c in H.CASES}
    missing = {k: v[:2] for k, v in H.config_keys().items() if k not in have}
    assert not missing, "configuration regimes without a GPU case in tests/head_cases.py: %r" % missing


def test_config_regimes_include_the_untested_geometry():
    """the C2 size puts every NT the README table runs on several, uneven tiles per CTA in both directions"""
    keys = H.config_keys()
    for nt in (1, 2, 4, 7, 8):
        for precision in ("bf16", "split"):
            assert ("fwd", nt, "several", "uneven", "whole", "within", "none", "no-bias", precision) in keys
            assert ("bwd", nt, "several", "uneven", "whole", "within", "vec", "no-dbias", precision) in keys
    assert ("bwd", 1, "several", "uneven", "whole", "within", "vec", "dbias", "split") in keys          # DynUNet


def test_table_covers_every_nt_edge_and_combination():
    cases = H.CASES
    for nt in range(1, 9):
        for precision in ("bf16", "split"):
            assert any(c.fwd_key[1] == nt and c.fwd_key[2] == "several" and c.bwd_key[2] == "several" and c.precision == precision
                       for c in cases), (nt, precision)
        lo, hi = (9 if nt == 1 else 16 * nt - 15), 16 * nt
        assert {lo, hi} <= {c.n_out for c in cases}, nt
    assert {c.c for c in cases} >= set(range(8, 65, 8))
    assert {(c.act, c.bias) for c in cases} == {(a, b) for a in H.ACTS for b in (False, True)}
    assert any(c.ld is not None for c in cases)
    assert {c.bwd_key[6] for c in cases} == {"vec", "scalar", "unaligned"}
    assert {c.fwd_key[2] for c in cases} == {"one", "several"} and {c.bwd_key[2] for c in cases} == {"one", "several"}
    assert {c.fwd_key[3] for c in cases} == {"even", "uneven"} and {c.bwd_key[3] for c in cases} == {"even", "uneven"}
    assert {c.fwd_key[4] for c in cases} == {"whole", "partial"} and {c.fwd_key[5] for c in cases} == {"within", "straddle"}
    assert any(c.geometry["kpad"] for c in cases) and any(not c.geometry["kpad"] for c in cases)
    assert any(c.geometry["wg1_dw"] for c in cases) and any(not c.geometry["wg1_dw"] for c in cases)
    # the offset rows: S % 4 == 0, so the aligned run they are compared with takes the vector path
    assert all(H.head_geometry(c.n_out, c.c, c.n, c.dims)["path"] == "vec" for c in cases if c.offset)


def test_case_ids_are_unique():
    ids = collections.Counter(c.id for c in H.CASES)
    assert max(ids.values()) == 1, [i for i, k in ids.items() if k > 1]
