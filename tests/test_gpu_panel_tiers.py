"""Exact-arithmetic parity of the tiered panel (PageRank, panel.cuh / build_panel_layout), edge for edge.

After tier 0 (the first LUXB_SB_BLOCKS hot source blocks over every hub), the remaining blocks of the hot set each
serve a prefix of the hubs ordered by in-degree: block b keeps the hubs whose expected edges from b reach
LUXB_SB_SLOT_EDGES.  LUXB_SB_TIER=1 forces the tiers; each case is compared with one oracle iteration from integer
inputs on which every summation order is exact (the method and helpers of test_gpu_exact.py), so a dropped,
duplicated or misrouted edge or partial changes the result.

Covered: tiers with prefixes shorter than the hub list and a block size that does not divide the hot set, prefixes
reaching 0 before the end of the hot set, a single tier block, every destination in every block, the tiers beside the
cold-hub stream at its segment cap (sort keys past 255), every panel shape, both fix-ups on a panel of more than 1024
fix-up blocks, and the default configuration at C1 and C2.  Also: two runs with the three-kernel fix-up give identical
values.  LUXB_SKIP_HEAVY=1 skips C2."""
import numpy as np
import pytest

import oracle as O
import lux_b200 as L
from graphs import in_degrees, rmat
from test_gpu_cold_split import cold_rule, segments
from test_gpu_exact import assert_bit_equal, exact_pr_inputs, exact_steps, graph, heavy, hot_set_size, set_env

pytestmark = pytest.mark.gpu


def run_tiers(name, env, monkeypatch, rounds=1):
    set_env(monkeypatch, dict(env, LUXB_SB=1, LUXB_SB_TIER=1))
    row_end, src = graph(name)
    with L.LuxGraph.from_csc(row_end, src) as g:
        g.init()
        st = g.stats()
        exact_steps(g, row_end, src, "%s %s" % (name, env), rounds)
    return st


# name: (graph, environment)
TIER_CASES = {
    "prefixes_bs_not_dividing_the_hot_set": ("rmat17", dict(LUXB_SB_BS=1000, LUXB_SB_BLOCKS=4, LUXB_SB_MIN_INDEG=16,
                                                            LUXB_SB_SLOT_EDGES=2)),
    "prefix_reaching_0": ("rmat16", dict(LUXB_SB_BS=512, LUXB_SB_BLOCKS=2, LUXB_SB_MIN_INDEG=8, LUXB_SB_SLOT_EDGES=40)),
    "single_tier_block": ("rmat16", dict(LUXB_SB_BS=4096, LUXB_SB_MIN_INDEG=8, LUXB_SB_SLOT_EDGES=0)),
    "every_destination_in_every_block": ("rmat16", dict(LUXB_SB_BS=2048, LUXB_SB_BLOCKS=2, LUXB_SB_MIN_INDEG=1,
                                                        LUXB_SB_SLOT_EDGES=0)),
    "beside_the_cold_hub_stream_at_its_cap": ("rmat16", dict(LUXB_CS=1, LUXB_CS_SEG_MB=4e-6, LUXB_HOT_MB=0.04, LUXB_SB_BS=128,
                                                             LUXB_SB_BLOCKS=8, LUXB_SB_MIN_INDEG=16, LUXB_SB_SLOT_EDGES=1)),
}


@pytest.mark.parametrize("panel_shape", range(6))
@pytest.mark.parametrize("case", sorted(TIER_CASES))
def test_tiers_every_panel_shape(case, panel_shape, monkeypatch):
    name, env = TIER_CASES[case]
    env = dict(env, LUXB_SEG_PANEL_SHAPE=panel_shape, LUXB_SEG_MAIN_SHAPE=(panel_shape + 2) % 8)
    row_end, src = graph(name)
    hot = hot_set_size(row_end, src, float(env.get("LUXB_HOT_MB", 24.0)))
    bs = env["LUXB_SB_BS"]
    nb_all = -(-hot // bs)
    if case == "single_tier_block":
        env["LUXB_SB_BLOCKS"] = nb_all - 1
    st = run_tiers(name, env, monkeypatch)
    nb0, nh = st["panel_blocks"], st["panel_hubs"]
    # the configuration is the one the case is named after
    assert st["panel_edges"] > 0 and nb0 == min(env["LUXB_SB_BLOCKS"], nb_all) and st["tier_edges"] > 0, (st, hot)
    assert st["tier_slots"] <= st["tier_blocks"] * nh
    if case == "prefixes_bs_not_dividing_the_hot_set":
        assert hot % bs != 0 and st["tier_slots"] < st["tier_blocks"] * nh, st
    elif case == "prefix_reaching_0":
        assert 0 < st["tier_blocks"] < nb_all - nb0, (st, nb_all)
    elif case == "single_tier_block":
        assert st["tier_blocks"] == 1 and st["tier_slots"] == nh, st
    elif case == "every_destination_in_every_block":
        assert nh == int((in_degrees(row_end) > 0).sum()) and st["tier_blocks"] == nb_all - nb0
        assert st["tier_slots"] == st["tier_blocks"] * nh
    elif case == "beside_the_cold_hub_stream_at_its_cap":
        n_cold = int(cold_rule(row_end, src, env["LUXB_HOT_MB"])[1].sum())
        assert n_cold > 255 - nb0 and st["cold_hub_segments"] == segments(n_cold, 1, nb0) and st["tier_blocks"] > 0, st
        assert nb0 + st["tier_blocks"] + st["cold_hub_segments"] > 256  # the sort keys need more than 8 bits


@pytest.mark.parametrize("fused", [0, 1])
def test_tiers_fixups_rmat24_several_rounds(fused, monkeypatch):
    """One tier-0 block and tier prefixes over the hubs of in-degree >= 64 put more than 2^27 of RMAT-24's 2^28 edges
    in the panel: with the 512-edge pieces of panel shape 0 that is more than 1024 fix-up blocks of 256 pieces.  Two
    rounds of set_values / iterate on one handle reuse the chained scan's status words."""
    set_env(monkeypatch, dict(LUXB_SB=1, LUXB_SB_TIER=1, LUXB_FUSED_FIXUP=fused, LUXB_SEG_PANEL_SHAPE=0, LUXB_SB_BLOCKS=1,
                              LUXB_SB_SLOT_EDGES=0.5))
    scale = 24
    row_end, src = rmat(scale)
    with L.LuxGraph.from_rmat(scale, 1 << scale, 16 << scale, 27) as g:
        g.init()
        st = g.stats()
        assert st["tier_blocks"] > 0 and (st["panel_edges"] + st["tier_edges"]) // 512 > 1024 * 256, st
        exact_steps(g, row_end, src, "rmat24 tiers fused=%d" % fused, rounds=2)


def test_tiers_default_c1(monkeypatch):
    monkeypatch.delenv("LUXB_SB_TIER", raising=False)
    nv, ne, seed = 7414866, 194109311, 1
    with L.LuxGraph.from_rmat(23, nv, ne, seed) as g:
        row_end, src = g.local_csc()
        g.init()
        st = g.stats()
        assert st["panel_edges"] > 0, st
        exact_steps(g, row_end, src, "C1 tiers %s" % st)


@heavy
def test_tiers_default_c2(monkeypatch):
    """RMAT-27 in the default configuration (the tiers are on), on the oracle generator's destination blocks."""
    monkeypatch.delenv("LUXB_SB_TIER", raising=False)
    scale, seed = 27, 27
    nv, ne = 1 << scale, 16 << scale
    block_shift = 14
    nb = nv >> block_shift
    sel = (np.random.default_rng(13).integers(0, 32, nb) == 0).astype(np.uint8)
    sel[0] = sel[1] = sel[nb - 1] = 1
    blk = O.rmat_blocks(scale, nv, ne, seed, block_shift, sel, want_deg=True)
    xs = exact_pr_inputs(nv, int(in_degrees(blk["row_end"]).max()), passes=3)
    with L.LuxGraph.from_rmat(scale, nv, ne, seed) as g:
        g.init()
        st = g.stats()
        assert st["panel_edges"] > 0 and st["tier_blocks"] > 0 and st["tier_edges"] > 0, st
        for i, x in enumerate(xs):
            g.set_values(x)
            g.iterate(1)
            assert_bit_equal(g.values()[blk["vid"]], O.pagerank_iter_compact(nv, blk, blk["deg"], x), "C2 tiers input %d" % i)


def test_tiers_values_run_to_run_identical(monkeypatch):
    """Three-kernel fix-up (fixed association): two handles give bit-identical values after several iterations."""
    set_env(monkeypatch, dict(LUXB_SB=1, LUXB_SB_TIER=1, LUXB_FUSED_FIXUP=0, LUXB_SB_BS=1000, LUXB_SB_BLOCKS=4,
                              LUXB_SB_MIN_INDEG=16, LUXB_SB_SLOT_EDGES=2))
    row_end, src = graph("rmat17")
    out = []
    for _ in range(2):
        with L.LuxGraph.from_csc(row_end, src) as g:
            g.init()
            assert g.stats()["tier_blocks"] > 0
            g.iterate(5)
            out.append(g.values())
    assert_bit_equal(out[0], out[1], "two runs")
