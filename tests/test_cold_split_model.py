"""Executable model (numpy, CPU) of the three-way split of a PageRank partition on one rank (lux_b200/csrc/api.cu
build_hot_layout / build_panel_layout, panel.cuh), checked against per-vertex sums computed directly from the CSC:

  * gather space Z = [hot copies | cold-active values (0 < out-degree < tau) in id order]; a source's gather id is its
    hot rank or H + its cold rank, and one gather over [hot order | cold list] refreshes all of Z    (build_hot_layout)
  * edge keys = source groups: (hot source of block b -> hub) = b, (cold source of segment s -> hub) = NB + s, the
    rest 511 (kSplitKeyMain); segments of `seg` values, raised so that S <= 255 - NB; one stable sort separates panel,
    cold-hub and main                                                                             (hub_key_kernel)
  * one table of groups: group g (block b = g, or segment s = g - NB) serves every hub here (no tiers) and owns the
    slots vbase[g] + h of one raw-partial array; the panel stream covers the slots of groups [0, NB), the cold-hub
    stream those of [NB, NB + S), its close list carrying slot numbers; main in-degree = in-degree minus the edges
    of both                                                              (group_fill_kernel, main_indeg_kernel)
  * each stream swept by the flagged-stream model of test_seg_model.py; hubs = main raw sum + panel partials in block
    order + cold partials in segment order, all read from that array                            (combine_hub_kernel)
Integer edge values make every summation order exact, so the comparison is bit-exact."""
import numpy as np
import pytest

import oracle as O
from graphs import in_degrees, rmat
from test_seg_model import direct_sums, run_model

CAP = 4096
KEY_MAIN = 511  # kSplitKeyMain


def hot_cold_layout(row_end, src, hot_mb):
    """(H, gather id per edge, Z source list [hot order | cold list])."""
    nv = len(row_end)
    deg = O.out_degree(nv, src).astype(np.int64)
    h_max = min(int(hot_mb * 1e6 / 4.0), nv)
    hist = np.bincount(np.minimum(deg, CAP), minlength=CAP + 1)
    above, tau = 0, CAP + 1
    for d in range(CAP, 1, -1):
        if above + int(hist[d]) > h_max:
            break
        above += int(hist[d])
        tau = d
    hot = deg >= tau
    hot_order = np.nonzero(hot)[0][np.argsort(-np.minimum(deg[hot], CAP), kind="stable")]
    cold = (deg > 0) & (deg < tau)
    cold_list = np.nonzero(cold)[0]
    gmap = np.zeros(nv, np.int64)
    gmap[cold_list] = len(hot_order) + np.arange(len(cold_list))
    gmap[hot_order] = np.arange(len(hot_order))
    assert not (deg[src] == 0).any()
    return len(hot_order), gmap[src], np.concatenate([hot_order, cold_list])


def split(row_end, gid, H, n_cold, min_indeg, bs, nb_max, seg_values):
    """Keys of every edge, block / segment counts, the group table and the three CSCs as
    {stream: (row_end, edge indices, first slot)}."""
    nv = len(row_end)
    indeg = in_degrees(row_end)
    dst = np.repeat(np.arange(nv), indeg)
    is_hub = indeg >= min_indeg
    hub_idx = np.cumsum(is_hub) - is_hub
    Nh = int(is_hub.sum())
    n_src = min(H, nb_max * bs)
    NB = -(-n_src // bs)
    s_max = 255 - NB
    seg = min(max(seg_values, -(-n_cold // s_max)), n_cold)
    S = -(-n_cold // seg)
    key = np.full(len(gid), KEY_MAIN, np.int64)
    hub_e = is_hub[dst]
    key[hub_e & (gid < n_src)] = gid[hub_e & (gid < n_src)] // bs
    c = hub_e & (gid >= H)
    key[c] = NB + (gid[c] - H) // seg
    assert key[key != KEY_MAIN].max(initial=0) < KEY_MAIN
    order = np.argsort(key, kind="stable")
    k_sorted = key[order]
    vbase = np.arange(NB + S + 1, dtype=np.int64) * Nh  # every group serves all Nh hubs
    streams = {}
    for name, lo, hi in (("panel", 0, NB), ("cold", NB, NB + S)):
        sel = order[(k_sorted >= lo) & (k_sorted < hi)]
        v = vbase[key[sel]] + hub_idx[dst[sel]]
        assert np.all(np.diff(v) >= 0)  # the stable sort leaves every slot's edges contiguous, in order
        v0 = int(vbase[lo])
        streams[name] = (np.cumsum(np.bincount(v - v0, minlength=int(vbase[hi]) - v0)).astype(np.uint64), sel, v0)
    main = order[k_sorted == KEY_MAIN]
    cov = np.bincount(dst[order[k_sorted != KEY_MAIN]], minlength=nv)
    streams["main"] = (np.cumsum(indeg - cov).astype(np.uint64), main, 0)
    return streams, NB, S, seg, vbase, is_hub


def sweep_and_combine(streams, vals, NB, S, vbase, is_hub, drop_last_segment=False):
    shape = dict(piece=16, rnd=8, stage=32)
    raw = {name: {v0 + v: x for v, x in run_model(re, vals[sel], **shape).items()} for name, (re, sel, v0) in streams.items()}
    assert not raw["panel"].keys() & raw["cold"].keys()
    partial = {**raw["panel"], **raw["cold"]}  # one array of (group, hub) slots
    out = dict(raw["main"])
    for h, v in enumerate(np.nonzero(is_hub)[0]):
        t = raw["main"].get(int(v), 0)
        for b in range(NB):
            t += partial.get(int(vbase[b]) + h, 0)
        for g in range(NB, NB + S - (1 if drop_last_segment else 0)):
            t += partial.get(int(vbase[g]) + h, 0)
        out[int(v)] = t
    return out


# (graph, hot set MB, hub min in-degree, panel block size, max blocks, cold segment values)
CASES = {
    "seg_not_dividing": ("rmat12", 0.004, 8, 256, 48, 100),
    "single_segment": ("rmat12", 0.004, 8, 256, 48, 1 << 30),
    "one_value_segments": ("rmat10", 24.0, 4, 64, 48, 1),
    "one_value_raised_to_the_cap": ("rmat12", 0.004, 8, 16, 64, 1),
    "every_vertex_a_hub": ("rmat12", 0.004, 1, 128, 48, 50),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_three_way_split(case):
    name, hot_mb, min_indeg, bs, nb_max, seg_values = CASES[case]
    row_end, src = rmat(int(name[len("rmat"):]))
    H, gid, zsrc = hot_cold_layout(row_end, src, hot_mb)
    n_cold = len(zsrc) - H
    streams, NB, S, seg, vbase, is_hub = split(row_end, gid, H, n_cold, min_indeg, bs, nb_max, seg_values)
    # every edge lands in exactly one stream
    all_e = np.concatenate([sel for _, sel, _ in streams.values()])
    assert len(all_e) == len(src) and np.array_equal(np.sort(all_e), np.arange(len(src)))
    for name_s, (re, sel, _) in streams.items():
        assert int(re[-1]) == len(sel), name_s
    assert S <= 255 - NB and NB + S < KEY_MAIN and len(streams["cold"][1]) > 0
    assert streams["cold"][2] == vbase[NB] and len(streams["cold"][0]) == vbase[NB + S] - vbase[NB]
    if case == "one_value_segments":
        assert S == n_cold
    if case == "one_value_raised_to_the_cap":
        assert n_cold > 255 - NB and S <= 255 - NB
    if case == "single_segment":
        assert S == 1
    if case == "seg_not_dividing":
        assert n_cold % seg_values and S > 1
    # the combine over (main raw + panel blocks + cold segments) equals the per-vertex sum, on integer values
    x = np.random.default_rng(3).integers(1, 1000, len(row_end)).astype(np.int64)
    vals = x[src]
    want = direct_sums(row_end, vals)
    assert sweep_and_combine(streams, vals, NB, S, vbase, is_hub) == want
    # and a missing cold-segment partial is seen
    in_last = (gid[streams["cold"][1]] - H) // seg == S - 1
    assert (sweep_and_combine(streams, vals, NB, S, vbase, is_hub, drop_last_segment=True) != want) == bool(in_last.any())


@pytest.mark.parametrize("hot_mb", [0.004, 24.0])
def test_compact_cold_index_round_trips(hot_mb):
    """Z = x[[hot order | cold list]] holds every source's value at its gather id, before and after a refresh."""
    row_end, src = rmat(12)
    H, gid, zsrc = hot_cold_layout(row_end, src, hot_mb)
    assert len(np.unique(zsrc)) == len(zsrc) and np.all(np.diff(zsrc[H:]) > 0)  # cold list: ascending ids
    rng = np.random.default_rng(1)
    for _ in range(2):  # values, then a refresh with other values
        x = rng.random(len(row_end)).astype(np.float32)
        Z = x[zsrc]
        assert np.array_equal(Z[gid].view(np.uint32), x[src].view(np.uint32))
