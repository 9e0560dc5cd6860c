"""Exact-arithmetic parity of the cold-hub stream (PageRank on one rank, panel.cuh ColdSplit), edge for edge.

Edges from a cold source (0 < out-degree < tau) into a hub move from the main stream into a third flagged stream over
virtual vertices (cold source segment s, hub h), and combine_hub_kernel adds their raw partials after the panel
partials.  LUXB_CS=1 forces the split; each case is compared with one oracle iteration from integer inputs on which
every summation order is exact (the method and helpers of test_gpu_exact.py), so a dropped, duplicated or misrouted
cold-hub edge or partial changes the result.

Covered: a segment size that does not divide the cold count, a single segment, one-value segments (below the sort
key's cap and raised to it), hubs without cold in-edges, every vertex a hub, the cold-hub stream in every main shape,
both fix-ups on a cold-hub stream of more than 1024 fix-up blocks, and the default configuration at C1 and C2 with the
split forced.  LUXB_SKIP_HEAVY=1 skips C2."""
import numpy as np
import pytest

import oracle as O
import lux_b200 as L
from graphs import in_degrees, rmat
from test_gpu_exact import assert_bit_equal, exact_pr_inputs, exact_steps, graph, heavy, set_env

pytestmark = pytest.mark.gpu


def cold_rule(row_end, src, hot_mb=24.0, cap=4096):
    """The hot / cold rule of build_hot_layout (lux_b200/csrc/api.cu): tau >= 2 the smallest threshold whose vertices
    of out-degree >= tau fit in hot_mb MB of values; cold = 0 < out-degree < tau.  Returns (H, cold mask)."""
    nv = len(row_end)
    deg = O.out_degree(nv, src)
    h_max = min(int(hot_mb * 1e6 / 4.0), nv)
    hist = np.bincount(np.minimum(deg, cap), minlength=cap + 1)
    above, tau = 0, cap + 1
    for d in range(cap, 1, -1):
        if above + int(hist[d]) > h_max:
            break
        above += int(hist[d])
        tau = d
    return above, (deg > 0) & (deg < tau)


def cold_hub_counts(row_end, src, cold, min_indeg):
    """Per hub (in-degree >= min_indeg): its cold in-edges."""
    indeg = in_degrees(row_end)
    dst = np.repeat(np.arange(len(row_end)), indeg)
    per_dst = np.bincount(dst[cold[src]], minlength=len(row_end))
    return per_dst[indeg >= min_indeg]


def run_cold(name, env, monkeypatch, rounds=1):
    set_env(monkeypatch, dict(env, LUXB_SB=1, LUXB_CS=1))
    row_end, src = graph(name)
    with L.LuxGraph.from_csc(row_end, src) as g:
        g.init()
        st = g.stats()
        assert st["cold_hub_edges"] > 0 and st["cold_hub_segments"] > 0, st
        exact_steps(g, row_end, src, "%s %s" % (name, env), rounds)
    return st


def segments(n_cold, seg_values, n_blocks):
    """Segment count the build chooses: seg_values per segment, raised so that n_blocks + S <= 255 (8-bit sort key)."""
    s_max = 255 - n_blocks
    seg = min(max(seg_values, -(-n_cold // s_max)), n_cold)
    return -(-n_cold // seg)


# name: (graph, environment); LUXB_CS_SEG_MB = values * 4e-6
COLD_CASES = {
    "seg_not_dividing_the_cold_count": ("rmat16", dict(LUXB_CS_SEG_MB=1000 * 4e-6, LUXB_SB_MIN_INDEG=16, LUXB_HOT_MB=0.04)),
    "single_segment": ("rmat16", dict(LUXB_CS_SEG_MB=1000, LUXB_SB_MIN_INDEG=16, LUXB_HOT_MB=0.04)),
    "one_value_segments": ("rmat10", dict(LUXB_CS_SEG_MB=4e-6, LUXB_SB_MIN_INDEG=4, LUXB_HOT_MB=24, LUXB_SB_BS=64)),
    "one_value_segments_raised_to_the_cap": ("rmat16", dict(LUXB_CS_SEG_MB=4e-6, LUXB_SB_MIN_INDEG=16, LUXB_HOT_MB=0.04)),
    "every_vertex_a_hub": ("rmat16", dict(LUXB_CS_SEG_MB=0.02, LUXB_SB_MIN_INDEG=1, LUXB_HOT_MB=0.04, LUXB_SB_BS=512)),
}


@pytest.mark.parametrize("case", sorted(COLD_CASES))
def test_cold_split_edges(case, monkeypatch):
    name, env = COLD_CASES[case]
    row_end, src = graph(name)
    hot, cold = cold_rule(row_end, src, env["LUXB_HOT_MB"])
    n_cold = int(cold.sum())
    seg_values = max(1, int(env["LUXB_CS_SEG_MB"] * 1e6 / 4.0))
    st = run_cold(name, env, monkeypatch)
    per_hub = cold_hub_counts(row_end, src, cold, env["LUXB_SB_MIN_INDEG"])
    # the configuration is the one the case is named after
    assert st["cold_hub_edges"] == int(per_hub.sum()), st
    assert st["cold_hub_segments"] == segments(n_cold, seg_values, st["panel_blocks"]), (st, n_cold)
    assert (per_hub == 0).any()  # hubs without cold in-edges: their cold partials stay 0
    if case == "seg_not_dividing_the_cold_count":
        assert n_cold % seg_values != 0 and st["cold_hub_segments"] > 1
    elif case == "single_segment":
        assert st["cold_hub_segments"] == 1
    elif case == "one_value_segments":
        assert st["cold_hub_segments"] == n_cold <= 255 - st["panel_blocks"]
    elif case == "one_value_segments_raised_to_the_cap":
        assert n_cold > 255 - st["panel_blocks"] and st["cold_hub_segments"] <= 255 - st["panel_blocks"]
    elif case == "every_vertex_a_hub":
        assert st["panel_hubs"] == int((in_degrees(row_end) > 0).sum())


@pytest.mark.parametrize("cs_shape", range(8))
def test_cold_split_every_main_shape(cs_shape, monkeypatch):
    """The cold-hub stream's kernel in every main shape (the main stream keeps another one)."""
    env = dict(LUXB_CS_SHAPE=cs_shape, LUXB_SEG_MAIN_SHAPE=(cs_shape + 3) % 8, LUXB_CS_SEG_MB=0.1, LUXB_SB_MIN_INDEG=8,
               LUXB_HOT_MB=0.2)
    for name in ("rmat16", "rmat17"):
        run_cold(name, env, monkeypatch)


@pytest.mark.parametrize("fused", [0, 1])
def test_cold_split_fixups_rmat23_several_rounds(fused, monkeypatch):
    """A hot set of about 2500 values (RMAT-23 has 2048 sources of out-degree >= 4096, where the rule's histogram
    stops) and every vertex a hub send most of RMAT-23's 2^27 edges through the cold-hub stream: with the 256-edge
    pieces of main shape 6 that is more than 1024 fix-up blocks of 256 pieces.  Three rounds
    of set_values / iterate on one handle reuse the chained scan's status words."""
    set_env(monkeypatch, dict(LUXB_SB=1, LUXB_CS=1, LUXB_FUSED_FIXUP=fused, LUXB_CS_SHAPE=6, LUXB_HOT_MB=0.01,
                              LUXB_SB_MIN_INDEG=1))
    scale = 23
    row_end, src = rmat(scale)
    with L.LuxGraph.from_rmat(scale, 1 << scale, 16 << scale, 27) as g:
        g.init()
        st = g.stats()
        assert -(-st["cold_hub_edges"] // 256) > 1024 * 256, st
        exact_steps(g, row_end, src, "rmat23 cold-hub fused=%d" % fused, rounds=3)


def test_cold_split_default_c1(monkeypatch):
    monkeypatch.setenv("LUXB_CS", "1")
    nv, ne, seed = 7414866, 194109311, 1
    with L.LuxGraph.from_rmat(23, nv, ne, seed) as g:
        row_end, src = g.local_csc()
        g.init()
        assert g.stats()["cold_hub_edges"] > 0
        exact_steps(g, row_end, src, "C1 cold-hub")


@heavy
def test_cold_split_default_c2(monkeypatch):
    """RMAT-27 in the default configuration with the split forced, on the oracle generator's destination blocks."""
    monkeypatch.setenv("LUXB_CS", "1")
    scale, seed = 27, 27
    nv, ne = 1 << scale, 16 << scale
    block_shift = 14
    nb = nv >> block_shift
    sel = (np.random.default_rng(11).integers(0, 32, nb) == 0).astype(np.uint8)
    sel[0] = sel[1] = sel[nb - 1] = 1
    blk = O.rmat_blocks(scale, nv, ne, seed, block_shift, sel, want_deg=True)
    xs = exact_pr_inputs(nv, int(in_degrees(blk["row_end"]).max()), passes=3)
    with L.LuxGraph.from_rmat(scale, nv, ne, seed) as g:
        g.init()
        st = g.stats()
        assert st["panel_edges"] > 0 and st["cold_hub_edges"] > 0, st
        for i, x in enumerate(xs):
            g.set_values(x)
            g.iterate(1)
            assert_bit_equal(g.values()[blk["vid"]], O.pagerank_iter_compact(nv, blk, blk["deg"], x), "C2 cold-hub input %d" % i)


def test_cold_split_values_run_to_run_identical(monkeypatch):
    """Three-kernel fix-up (fixed association): two handles give bit-identical values after several iterations."""
    set_env(monkeypatch, dict(LUXB_SB=1, LUXB_CS=1, LUXB_FUSED_FIXUP=0, LUXB_CS_SEG_MB=0.1, LUXB_HOT_MB=0.2, LUXB_SB_MIN_INDEG=8))
    row_end, src = graph("rmat17")
    out = []
    for _ in range(2):
        with L.LuxGraph.from_csc(row_end, src) as g:
            g.init()
            g.iterate(5)
            out.append(g.values())
    assert_bit_equal(out[0], out[1], "two runs")
