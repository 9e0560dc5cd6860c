"""The wide exact-input method of tests/test_gpu_wide_exact.py, proved on the CPU with the oracle alone.

The inputs of graphs.exact_pr_inputs / exact_cf_inputs keep every vertex sum below 2^21 (PageRank) or 2^22 (CF).  There
fp32 is exact in any order, so a sweep whose fp64 carry or combine had been narrowed to fp32 would still match the
oracle bit for bit: those inputs pin which edge lands where, not the width of the arithmetic.  The inputs of
wide_inputs.wide_exact_pr_inputs / wide_exact_cf_inputs keep every fp32 unit of a sweep exact while the vertex sums pass
2^25.  Here a numpy model of the device's units (fp32 sums of a piece, a round, a panel slot or a CF chunk, combined in
fp64 and narrowed once) equals the oracle bit for bit on them, the same model with one step narrowed to fp32 does
not, and on the narrow inputs every variant agrees with the oracle.  The update is applied by the oracle itself
(`apply_update`), so the comparison is with O.pagerank_iter's own fma and division."""
import numpy as np

import oracle as O
from graphs import exact_cf_inputs, exact_pr_inputs, in_degrees, rmat
from wide_inputs import (WIDE_MIN, regular_indegree, tier0_panel, vertex_sums, wide_exact_cf_inputs, wide_exact_pr_inputs,
                         wide_vertices)

CF_GAMMA = np.float32(0.00000035)
PIECE = 1024  # the longest piece of the main flagged-stream shapes (shape 3: 4 rounds of 256 edges)
ROUND = 256


def f32_chain(parts, owner, n):
    """Per owner, its parts added in order with a float32 rounding after every add (a narrowed carry / combine)."""
    order = np.argsort(owner, kind="stable")
    parts, owner = parts[order], owner[order]
    first = np.searchsorted(owner, owner, side="left")
    pos = np.arange(len(owner)) - first
    acc = np.zeros(n, np.float32)
    for k in range(int(pos.max()) + 1 if len(pos) else 0):
        sel = pos == k
        acc[owner[sel]] = (acc[owner[sel]].astype(np.float64) + parts[sel]).astype(np.float32)
    return acc


def unit_partials(row_end, x, src, unit):
    """fp64 sums (exact: integers) of the runs of a vertex's in-edges inside one `unit`-edge window of the CSC order
    (the flagged stream of the plain sweep is the CSC order from word 0): (partial, vertex) per (vertex, window)."""
    nv, ne = len(row_end), len(src)
    dst = np.repeat(np.arange(nv), in_degrees(row_end))
    key = dst.astype(np.int64) * (ne // unit + 1) + np.arange(ne) // unit
    starts = np.nonzero(np.concatenate([[True], key[1:] != key[:-1]]))[0]
    return np.add.reduceat(x[src].astype(np.float64), starts), dst[starts]


def apply_update(deg, acc):
    """update(acc) per vertex by the oracle: each vertex gets one in-edge from itself, whose value is acc."""
    nv = len(deg)
    return O.pagerank_iter(np.arange(1, nv + 1, dtype=np.uint64), np.arange(nv, dtype=np.uint32), deg, acc.astype(np.float32))


def pr_models(row_end, src, x, piece=PIECE, rnd=ROUND):
    """Stored values of one PageRank step under the device's arithmetic and under each narrowed variant."""
    nv = len(row_end)
    deg = O.out_degree(nv, src)
    pp, pv = unit_partials(row_end, x, src, piece)
    split = np.bincount(pv, minlength=nv)[pv] > 1  # a vertex in one piece is narrowed once, from its whole sum
    assert np.all(pp[split] < (1 << 24)), "a piece partial of a vertex over several pieces is not exact in fp32"
    out = {"device": apply_update(deg, np.bincount(pv, weights=pp, minlength=nv).astype(np.float32)),
           "cross_piece_combine_fp32": apply_update(deg, f32_chain(pp, pv, nv))}
    # the round-to-round carry inside a piece in fp32, then pieces in fp64
    rp, rv = unit_partials(row_end, x, src, rnd)
    ne = len(src)
    dst = np.repeat(np.arange(nv), in_degrees(row_end))
    piece_of = np.arange(ne) // piece
    starts = np.nonzero(np.concatenate([[True], (dst[1:] != dst[:-1]) | ((np.arange(1, ne) // rnd) != (np.arange(ne - 1) // rnd))]))[0]
    seg = dst[starts].astype(np.int64) * (ne // piece + 1) + piece_of[starts]
    uniq, seg_id = np.unique(seg, return_inverse=True)
    per_piece = f32_chain(rp, seg_id, len(uniq)).astype(np.float64)
    out["round_carry_fp32"] = apply_update(deg, np.bincount((uniq // (ne // piece + 1)).astype(np.int64), weights=per_piece,
                                                            minlength=nv).astype(np.float32))
    return out


def check_wide(row_end, src, x, models, min_wide, narrowed):
    deg = O.out_degree(len(row_end), src)
    ref = O.pagerank_iter(row_end, src, deg, x)
    assert int(wide_vertices(vertex_sums(row_end, src, x)).sum()) >= min_wide
    assert np.array_equal(models["device"].view(np.uint32), ref.view(np.uint32))
    for name in narrowed:
        moved = int((models[name].view(np.uint32) != ref.view(np.uint32)).sum())
        assert moved >= max(1, min_wide // 4), "%s moves %d values" % (name, moved)


def check_narrow_inputs_blind(row_end, src, models_of):
    """On the narrow exact inputs every model, narrowed or not, is the oracle bit for bit: the gap this closes."""
    deg = O.out_degree(len(row_end), src)
    for x in exact_pr_inputs(len(row_end), int(in_degrees(row_end).max())):
        ref = O.pagerank_iter(row_end, src, deg, x)
        for name, got in models_of(x).items():
            assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), name


def star_in(n_leaves):
    """Vertex 0 with n_leaves in-edges from 1 .. n_leaves (in-degree 2^20: 1024 pieces of 1024 edges)."""
    return O.edges_to_csc(n_leaves + 1, np.arange(1, n_leaves + 1), np.zeros(n_leaves, np.int64))


# ---- the plain flagged stream: pieces and rounds ---------------------------------------------------------------------
def test_cross_piece_combine_star_and_rmat17():
    """A 2^20-leaf hub (one wide vertex over 1024 pieces) and RMAT-17, whose hubs span pieces: the fp64 fix-up is the
    oracle, an fp32 one is not.  Values up to K = 16383 (mean 8192) take a sum past 2^25 from about 4096 in-edges on:
    RMAT-17 has about a dozen such vertices, and at least 8 wide ones are asserted."""
    for (row_end, src), min_wide in ((star_in(1 << 20), 1), (rmat(17), 8)):
        x = wide_exact_pr_inputs(len(row_end), PIECE)
        check_wide(row_end, src, x, pr_models(row_end, src, x), min_wide, ["cross_piece_combine_fp32"])
        check_narrow_inputs_blind(row_end, src, lambda x: pr_models(row_end, src, x))


def test_round_carry_one_vertex_per_piece():
    """2048 vertices of in-degree 1024: with 1024-edge pieces of four 256-edge rounds each vertex is one piece, so its
    sum is the fp64 carry over four rounds, narrowed once.  Values up to K = 65535 keep each round exact and put half the
    sums past 2^25 (mean S = 2^25): at least 500 wide vertices; an fp32 carry rounds three times more."""
    row_end, src = regular_indegree(2048, PIECE)
    x = wide_exact_pr_inputs(len(row_end), ROUND)
    models = pr_models(row_end, src, x)
    check_wide(row_end, src, x, {"device": models["device"], "round_carry_fp32": models["round_carry_fp32"]}, 500,
               ["round_carry_fp32"])
    check_narrow_inputs_blind(row_end, src, lambda x: {k: v for k, v in pr_models(row_end, src, x).items() if k != "cross_piece_combine_fp32"})


# ---- the panel split: main part + slot partials of a hub ---------------------------------------------------------------
def panel_models(row_end, src, x, bs, blocks, min_indeg):
    """Hub v = main part (its edges from sources outside tier 0) then one partial per tier-0 source block, in block
    order (combine_hub_kernel); non-hubs are their own main part."""
    nv = len(row_end)
    deg = O.out_degree(nv, src)
    blk, _ = tier0_panel(row_end, src, bs, blocks, min_indeg)
    indeg = in_degrees(row_end)
    dst = np.repeat(np.arange(nv), indeg)
    hub = indeg[dst] >= min_indeg
    group = np.where(hub, blk[src] + 1, 0)  # 0: the main part
    key = dst.astype(np.int64) * (blocks + 1) + group
    o = np.argsort(key, kind="stable")
    k2 = key[o]
    starts = np.nonzero(np.concatenate([[True], k2[1:] != k2[:-1]]))[0]
    parts = np.add.reduceat(x[src[o]].astype(np.float64), starts)
    owner = dst[o][starts]
    assert np.all(parts < (1 << 24)), "a slot or main part is not exact in fp32"
    return {"device": apply_update(deg, np.bincount(owner, weights=parts, minlength=nv).astype(np.float32)),
            "slot_combine_fp32": apply_update(deg, f32_chain(parts, owner, nv))}


def test_slot_combine_tier0():
    """32768 vertices of in-degree 256 from uniform sources (every vertex a hub at in-degree >= 16), blocks of 512
    values, 48 blocks: tier-0 sources get values up to K = (2^24 - 1) / (most edges of one slot), the rest 1, so every
    slot, every hub's main part and every non-hub sums exactly.  On RMAT the top hub's largest slot alone nears 2^24,
    so its sums barely pass it; here a slot holds about 4 edges and a hub adds 48 of them, so most hubs are wide: at
    least 10 000 are asserted."""
    row_end, src = regular_indegree(32768, 256)
    bs, blocks, min_indeg = 512, 48, 16
    blk, most = tier0_panel(row_end, src, bs, blocks, min_indeg)
    x = wide_exact_pr_inputs(len(row_end), max(most, min_indeg), wide=blk >= 0)
    models = panel_models(row_end, src, x, bs, blocks, min_indeg)
    check_wide(row_end, src, x, models, 10000, ["slot_combine_fp32"])
    check_narrow_inputs_blind(row_end, src, lambda x: panel_models(row_end, src, x, bs, blocks, min_indeg))


# ---- collaborative filtering: chunk partials --------------------------------------------------------------------------
def cf_models(row_end, src, w, x, users):
    """Items' factors 10-19 (= rn(GAMMA * rn32(acc)): x_v is 0 there) from 256-edge chunk partials combined in fp64,
    and in fp32 after every add; and the exact accumulators."""
    nv = len(row_end)
    indeg = in_degrees(row_end)
    dst = np.repeat(np.arange(nv), indeg)
    xs = x[src].astype(np.float64)
    err = w.astype(np.float64) - (xs * x[dst].astype(np.float64)).sum(axis=1)
    first = np.concatenate([[0], row_end[:-1]]).astype(np.int64)
    chunk = dst.astype(np.int64) * (int(indeg.max()) // 256 + 1) + (np.arange(len(src)) - first[dst]) // 256
    starts = np.nonzero(np.concatenate([[True], chunk[1:] != chunk[:-1]]))[0]
    parts = np.add.reduceat(err[:, None] * xs[:, 10:], starts, axis=0)
    assert np.all(np.abs(parts) < (1 << 24)), "a chunk partial is not exact in fp32"
    owner = dst[starts]
    acc = np.stack([np.bincount(owner, weights=parts[:, f], minlength=nv) for f in range(10)], axis=1)
    narrowed = np.stack([f32_chain(parts[:, f], owner, nv) for f in range(10)], axis=1)
    out = {"device": CF_GAMMA * acc.astype(np.float32), "chunk_combine_fp32": CF_GAMMA * narrowed}
    return {k: v[users:] for k, v in out.items()}, acc[users:]


def test_cf_chunk_combine_hub_items():
    """20 000 users, 300 items, 1.5 M ratings (5 000 per item on average, over 20 chunks): the generator's item
    popularity is skewed, and about 60 % of the items' exact-factor accumulators are wide (at least half are
    asserted); an fp32 chunk combine moves at least a quarter of all of them."""
    users, items = 20000, 300
    row_end, src, w = O.gen_bipartite_csc(users, items, 1500000, 5)
    x = wide_exact_cf_inputs(users, items)
    ref = O.cf_iter(row_end, src, w, x)[users:, 10:]
    models, acc = cf_models(row_end, src, w, x, users)
    wide = (np.abs(acc) >= WIDE_MIN) & (acc != acc.astype(np.float32))
    assert wide.sum() >= 0.5 * wide.size
    assert np.array_equal(models["device"].view(np.uint32), ref.view(np.uint32))
    assert (models["chunk_combine_fp32"].view(np.uint32) != ref.view(np.uint32)).sum() >= 0.25 * ref.size
    # the narrow inputs: both combines are the oracle
    xn = exact_cf_inputs(users, items, int(in_degrees(row_end)[users:].max()))
    refn = O.cf_iter(row_end, src, w, xn)[users:, 10:]
    for name, got in cf_models(row_end, src, w, xn, users)[0].items():
        assert np.array_equal(got.view(np.uint32), refn.view(np.uint32)), name
