"""Executable model (numpy, CPU) of the tiered panel of a PageRank partition (lux_b200/csrc/api.cu build_panel_layout,
panel.cuh), checked against per-vertex sums computed directly from the CSC:

  * hubs (in-degree >= D) ordered by in-degree, descending, ties by ascending id        (hub_order_key_kernel + sort)
  * hub prefix N_b of every hot source block, from the histogram of one keying with every block over every hub: all
    hubs for the first nb0 blocks (tier 0); for a later block b, the hubs of in-degree d with d * m_b >= K, m_b =
    (edges block b -> hubs) / (edges into hubs), capped by N_{b-1}; trailing blocks with N_b = 0 are dropped; the
    edges are keyed again only when a prefix changed                                    (build_panel_layout)
  * edge keys: (hot source of block b -> hub h < N_b) = b, the rest main; a stable sort by hub position, then one by
    key, lists every block's edges by slot vbase[b] + h (vbase[b] = sum of N_b' for b' < b) and the main edges in CSC
    order; main in-degree = in-degree minus the panel coverage                     (hub_key_kernel, group_fill_kernel)
  * each stream swept by the flagged-stream model of test_seg_model.py; hubs = main raw sum + the partials of blocks
    b = 0, 1, ... while h < N_b                                                        (combine_hub_kernel)
Integer edge values make every summation order exact, so the comparison is bit-exact."""
import numpy as np
import pytest

from graphs import in_degrees, rmat
from test_cold_split_model import hot_cold_layout
from test_seg_model import direct_sums, run_model


def hub_order(indeg, min_indeg):
    hubs = np.nonzero(indeg >= min_indeg)[0]
    return hubs[np.argsort(-indeg[hubs], kind="stable")]


def tier_prefixes(hub_deg, block_hub_edges, nb0, slot_edges):
    """N_b for every block.  hub_deg: in-degrees of the ordered hubs; block_hub_edges[b]: edges block b -> any hub."""
    nh = len(hub_deg)
    e_hub = int(hub_deg.sum())
    pref = [nh] * len(block_hub_edges)
    for b in range(nb0, len(pref)):
        keep = 0
        if block_hub_edges[b] > 0:
            d_min = slot_edges * float(e_hub) / float(block_hub_edges[b])
            keep = int((hub_deg.astype(np.float64) >= d_min).sum())
        pref[b] = min(keep, pref[b - 1])
    while len(pref) > nb0 and pref[-1] == 0:
        pref.pop()
    return pref


def tiered_split(row_end, gid, H, min_indeg, bs, nb0, slot_edges):
    """The panel / main CSCs as {stream: (row_end, edge indices)}, the prefixes and the ordered hubs."""
    nv = len(row_end)
    indeg = in_degrees(row_end)
    dst = np.repeat(np.arange(nv), indeg)
    hubs = hub_order(indeg, min_indeg)
    pos = np.full(nv, -1, np.int64)
    pos[hubs] = np.arange(len(hubs))
    nb_all = -(-H // bs)
    hot_hub = (pos[dst] >= 0) & (gid < H)
    first = np.bincount(gid[hot_hub] // bs, minlength=nb_all)  # the first keying: every block over every hub
    pref = tier_prefixes(indeg[hubs], first, nb0, slot_edges)
    NB = len(pref)
    vbase = np.concatenate([[0], np.cumsum(pref)]).astype(np.int64)
    n_src = min(H, NB * bs)
    key = np.full(len(gid), -1, np.int64)
    cand = (pos[dst] >= 0) & (gid < n_src)
    b_of = gid // bs
    take = cand.copy()
    take[cand] = pos[dst[cand]] < np.asarray(pref, np.int64)[b_of[cand]]
    key[take] = b_of[take]
    # two stable sorts: by hub position (main edges count as position 0), then by key
    by_pos = np.argsort(np.where(take, pos[dst], 0), kind="stable")
    order = by_pos[np.argsort(np.where(key < 0, NB, key)[by_pos], kind="stable")]
    sel = order[: int(take.sum())]
    v = vbase[key[sel]] + pos[dst[sel]]
    assert np.all(np.diff(v) >= 0)  # the stable sort leaves every virtual vertex's edges contiguous, in order
    streams = {"panel": (np.cumsum(np.bincount(v, minlength=int(vbase[-1]))).astype(np.uint64), sel)}
    main = order[int(take.sum()):]
    cov = np.bincount(dst[sel], minlength=nv)
    streams["main"] = (np.cumsum(indeg - cov).astype(np.uint64), main)
    return streams, pref, vbase, hubs


def sweep_and_combine(streams, vals, pref, vbase, hubs, stop_early=False):
    shape = dict(piece=16, rnd=8, stage=32)
    blocks = [(int(vbase[b]), int(vbase[b + 1])) for b in range(len(pref))]
    raw = {"main": run_model(*streams["main"][:1], vals[streams["main"][1]], **shape),
           "panel": run_model(streams["panel"][0], vals[streams["panel"][1]], blocks=blocks, **shape)}
    out = dict(raw["main"])
    for h, v in enumerate(hubs):
        t = raw["main"].get(int(v), 0)
        b = 0
        while b < len(pref) - (1 if stop_early else 0) and h < pref[b]:
            t += raw["panel"].get(int(vbase[b]) + h, 0)
            b += 1
        out[int(v)] = t
    return out


# (graph, hot set MB, hub min in-degree, block size, tier-0 blocks, expected edges per slot)
CASES = {
    "tiers": ("rmat12", 24.0, 4, 64, 4, 2.0),
    "prefix_reaches_zero": ("rmat12", 24.0, 4, 64, 2, 40.0),
    "every_destination_in_every_block": ("rmat10", 24.0, 1, 32, 1, 0.0),
    "bs_not_dividing_the_hot_set": ("rmat12", 24.0, 8, 100, 3, 1.0),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_tiered_split(case):
    name, hot_mb, min_indeg, bs, nb0, slot_edges = CASES[case]
    row_end, src = rmat(int(name[len("rmat"):]))
    H, gid, _ = hot_cold_layout(row_end, src, hot_mb)
    streams, pref, vbase, hubs = tiered_split(row_end, gid, H, min_indeg, bs, nb0, slot_edges)
    indeg = in_degrees(row_end)
    nb_all = -(-H // bs)
    # hub order: in-degree descending, ties by id
    d = indeg[hubs]
    assert np.all((d[:-1] > d[1:]) | ((d[:-1] == d[1:]) & (hubs[:-1] < hubs[1:])))
    # prefixes: tier 0 over all hubs, then not increasing, no trailing empty block
    assert pref[:nb0] == [len(hubs)] * min(nb0, nb_all)
    assert all(a >= b for a, b in zip(pref, pref[1:])) and (len(pref) <= nb0 or pref[-1] > 0)
    # every edge lands in exactly one stream
    all_e = np.concatenate([sel for _, sel in streams.values()])
    assert len(all_e) == len(src) and np.array_equal(np.sort(all_e), np.arange(len(src)))
    if case == "tiers":
        assert len(pref) > nb0 and 0 < pref[-1] < len(hubs)
    elif case == "prefix_reaches_zero":
        assert nb0 < len(pref) < nb_all
    elif case == "every_destination_in_every_block":
        assert pref == [len(hubs)] * nb_all and len(hubs) == int((indeg > 0).sum())
    elif case == "bs_not_dividing_the_hot_set":
        assert H % bs != 0 and len(pref) == nb_all
    # the combine over (main raw + the blocks whose prefix holds the hub) equals the per-vertex sum, on integer values
    x = np.random.default_rng(4).integers(1, 1000, len(row_end)).astype(np.int64)
    vals = x[src]
    want = direct_sums(row_end, vals)
    assert sweep_and_combine(streams, vals, pref, vbase, hubs) == want
    # and a combine that stops one block early is seen
    last = len(pref) - 1
    last_edges = streams["panel"][0][vbase[last + 1] - 1] - (streams["panel"][0][vbase[last] - 1] if vbase[last] else 0)
    assert (sweep_and_combine(streams, vals, pref, vbase, hubs, stop_early=True) != want) == bool(last_edges > 0)
