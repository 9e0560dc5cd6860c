"""CPU model of the compact (group, hub) slot numbering of the source-blocked split (panel.cuh, seg.cuh).

Only the (source group, hub) pairs with at least one edge get a slot, numbered groups ascending, hubs ascending.  The
device keeps no close list for the group streams: per piece t it stores slot0 and the real range [lo, end) of its
heads (piece_slot_kernel), and the combine finds the slot of (g, h) as pre[w] + popc(bits[w] & lanes below h) in the
slot bitmap (slot_bits_kernel + an exclusive scan of the popcounts).  This module restates those rules in numpy and
holds them to the dense numbering they replace (close list of dense slots vbase[g] + h, dummies for the pads; the
combine over every dense slot, identity for the empty ones) on random incidences, the corner cases named in each test
included."""
import numpy as np
import pytest

DUMMY = -1


def layout(n_pref, counts):
    """Dense pair bases vbase, bitmap word bases wbase, the bitmap and its per-word exclusive prefix of set bits."""
    vbase = np.concatenate([[0], np.cumsum(n_pref)]).astype(np.int64)
    wbase = np.concatenate([[0], np.cumsum([(n + 31) // 32 for n in n_pref])]).astype(np.int64)
    bits = np.zeros(int(wbase[-1]), np.uint64)
    for g, n in enumerate(n_pref):
        for h in range(n):
            if counts[vbase[g] + h]:
                bits[wbase[g] + h // 32] |= np.uint64(1 << (h % 32))
    popc = np.array([bin(int(b)).count("1") for b in bits], np.int64)
    pre = np.concatenate([[0], np.cumsum(popc)])[:-1] if len(bits) else np.zeros(0, np.int64)
    return vbase, wbase, bits, pre


def compact_of_dense(counts):
    """compact slot of every dense pair (-1: no edges) = rank among the non-empty pairs"""
    ne = counts > 0
    return np.where(ne, np.cumsum(ne) - 1, -1)


def build_stream(counts, vbase, groups, per_group_blocks, stage, piece):
    """The flagged stream of groups `groups` (build_seg_stream): head flags per word, the dense close list (compact slot
    or DUMMY per head), tile_v, and the per-piece (slot0, lo, end) of piece_slot_kernel."""
    comp = compact_of_dense(counts)
    v0, v1 = vbase[groups[0]], vbase[groups[-1] + 1]
    blocks = [(vbase[g], vbase[g + 1]) for g in groups] if per_group_blocks else [(v0, v1)]
    heads, close = [], [DUMMY]  # close[J] = what head J closes; head 0 closes nothing
    wbase, hshift, rank_at = [], [], []
    pads_total = 0
    seg_before = 0
    for a, b in blocks:
        wbase.append(len(heads))
        hshift.append(pads_total)
        rank_at.append(seg_before)
        eb = int(counts[a:b].sum())
        for v in range(a, b):
            c = int(counts[v])
            if c:
                heads.extend([True] + [False] * (c - 1))
                seg_before += 1
        pad = stage - eb % stage
        heads.extend([True] * pad)
        pads_total += pad
    rank_at.append(seg_before)
    # the dense close list, as stream_heads_kernel writes it
    n_heads = sum(heads)
    close = np.full(n_heads + 1, DUMMY, np.int64)
    for bi, (a, b) in enumerate(blocks):
        r = rank_at[bi]
        for v in range(a, b):
            if counts[v]:
                close[1 + r + hshift[bi]] = comp[v]
                r += 1
    heads = np.array(heads)
    n_pieces = len(heads) // piece
    assert len(heads) % piece == 0
    tile_v = np.concatenate([[0], np.cumsum(heads.reshape(n_pieces, piece).sum(1))])
    slot_base = int((counts[:v0] > 0).sum())  # the cold-hub slots follow the panel's
    ps = []
    for t in range(n_pieces):
        b = max(i for i in range(len(blocks)) if wbase[i] <= t * piece)
        r0, r1 = rank_at[b], rank_at[b + 1]
        hb = r0 + hshift[b]
        i0, i1 = tile_v[t], tile_v[t + 1]
        last = min(i1, hb + 1 + (r1 - r0))
        ps.append((slot_base + i0 - 1 - hshift[b], int(i0 == hb), max(0, last - i0)))
    return heads, close, tile_v, ps


def check_stream(heads, close, tile_v, ps):
    n_real = 0
    for t, (slot0, lo, end) in enumerate(ps):
        for k, j in enumerate(range(tile_v[t], tile_v[t + 1])):
            real = lo <= k < end
            assert real == (close[j] != DUMMY), (t, k, j)
            if real:
                assert slot0 + k == close[j], (t, k, slot0, close[j])
                n_real += 1
    return n_real


def combine_dense(h, raw0, n_pref, n_blocks, vbase, dense):
    t = float(raw0)
    for b in range(n_blocks):
        if h >= n_pref[b]:
            break
        t += float(dense[vbase[b] + h])
    for k in range(n_blocks, len(n_pref)):
        t += float(dense[vbase[k] + h])
    return t


def combine_compact(h, raw0, n_pref, n_blocks, wbase, bits, pre, partial):
    t = float(raw0)
    w, me = h >> 5, 1 << (h & 31)
    order = [b for b in range(n_blocks) if h < n_pref[b]] + list(range(n_blocks, len(n_pref)))
    for g in order:
        wd = int(bits[wbase[g] + w])
        if wd & me:
            t += float(partial[pre[wbase[g] + w] + bin(wd & (me - 1)).count("1")])
    return t


def random_case(rng, nh, n_blocks, n_cold, density, empty_groups=(), dead_hubs=()):
    n_pref = [nh]
    for _ in range(1, n_blocks):
        n_pref.append(int(rng.integers(0, n_pref[-1] + 1)))
    n_pref += [nh] * n_cold
    vbase = np.concatenate([[0], np.cumsum(n_pref)])
    counts = np.where(rng.random(vbase[-1]) < density, rng.integers(1, 40, vbase[-1]), 0)
    for g in empty_groups:
        counts[vbase[g]:vbase[g + 1]] = 0
    for h in dead_hubs:
        for g in range(len(n_pref)):
            if h < n_pref[g]:
                counts[vbase[g] + h] = 0
    return n_pref, counts


CASES = {
    # name: (hubs, panel blocks, cold segments, density, empty groups, hubs empty in every group, stage, piece)
    "plain": (100, 6, 3, 0.4, (), (), 64, 16),
    "hubs_not_a_multiple_of_32": (77, 5, 2, 0.5, (), (), 32, 8),
    "sparse_tiers": (300, 9, 0, 0.03, (), (), 64, 32),
    "empty_groups": (70, 6, 3, 0.4, (0, 3, 7), (), 64, 16),
    "hub_empty_everywhere": (65, 4, 2, 0.6, (), (0, 31, 32, 64), 32, 16),
    "one_piece_per_stage": (40, 3, 2, 0.7, (), (), 16, 16),
    "all_empty_but_one": (50, 4, 1, 0.0, (), (), 32, 8),
}


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("case", sorted(CASES))
def test_compact_numbering_matches_the_dense_close_lists(case, seed):
    nh, nb, ncold, density, empty, dead, stage, piece = CASES[case]
    rng = np.random.default_rng(1000 * seed + len(case))
    n_pref, counts = random_case(rng, nh, nb, ncold, density, empty, dead)
    if case == "all_empty_but_one":
        counts[rng.integers(0, len(counts))] = 3
    vbase, wbase, bits, pre = layout(n_pref, counts)
    comp = compact_of_dense(counts)
    # bitmap + prefix give every non-empty pair its compact slot; gbase[g] = pre[wbase[g]]
    for g, n in enumerate(n_pref):
        for h in range(n):
            wd = int(bits[wbase[g] + h // 32])
            assert bool((wd >> (h % 32)) & 1) == bool(counts[vbase[g] + h])
            if counts[vbase[g] + h]:
                assert pre[wbase[g] + h // 32] + bin(wd & ((1 << (h % 32)) - 1)).count("1") == comp[vbase[g] + h]
        if n % 32:
            assert int(bits[wbase[g + 1] - 1]) >> (n % 32) == 0  # bits past N_g stay clear
    # the two streams: panel (one block per group), cold-hub (one block); their heads close the slots in order
    total = 0
    panel = list(range(nb))
    streams = [(panel, True)] + ([(list(range(nb, nb + ncold)), False)] if ncold else [])
    for groups, per_group in streams:
        heads, close, tile_v, ps = build_stream(counts, vbase, groups, per_group, stage, piece)
        total += check_stream(heads, close, tile_v, ps)
    assert total == int((counts > 0).sum())


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("case", sorted(CASES))
def test_combine_walk_equals_the_dense_walk(case, seed):
    nh, nb, ncold, density, empty, dead, _, _ = CASES[case]
    rng = np.random.default_rng(7 + 100 * seed + len(case))
    n_pref, counts = random_case(rng, nh, nb, ncold, density, empty, dead)
    vbase, wbase, bits, pre = layout(n_pref, counts)
    comp = compact_of_dense(counts)
    # partials on a 2^-40 grid with spread exponents: the fp64 sums round, so the association order shows
    vals = rng.random(len(counts)) * 2.0 ** rng.integers(-30, 30, len(counts))
    dense = np.where(counts > 0, vals, 0.0)  # empty dense slots hold the identity
    partial = np.zeros(int((counts > 0).sum()))
    partial[comp[counts > 0]] = vals[counts > 0]
    for h in range(nh):
        raw0 = rng.random()
        want = combine_dense(h, raw0, n_pref, nb, vbase, dense)
        got = combine_compact(h, raw0, n_pref, nb, wbase, bits, pre, partial)
        assert np.float64(got).view(np.uint64) == np.float64(want).view(np.uint64), (h, got, want)


def test_model_catches_the_mutations():
    """The rules above reject: a slot off by one at a piece's first entry, a real count one short, the prefix of the
    next word, the bitmap word of another group."""
    rng = np.random.default_rng(3)
    n_pref, counts = random_case(rng, 90, 5, 2, 0.5)
    vbase, wbase, bits, pre = layout(n_pref, counts)
    heads, close, tile_v, ps = build_stream(counts, vbase, list(range(5)), True, 64, 16)
    t = next(i for i, (s0, lo, end) in enumerate(ps) if lo == 0 and end > 1)
    for bad in [(ps[t][0] + 1, ps[t][1], ps[t][2]), (ps[t][0], ps[t][1], ps[t][2] - 1)]:
        mutated = list(ps)
        mutated[t] = bad
        with pytest.raises(AssertionError):
            check_stream(heads, close, tile_v, mutated)
    comp = compact_of_dense(counts)
    vals = rng.random(len(counts)) + 1.0
    dense = np.where(counts > 0, vals, 0.0)
    partial = np.zeros(int((counts > 0).sum()))
    partial[comp[counts > 0]] = vals[counts > 0]
    pre_next = np.concatenate([pre[1:], [pre[-1]]])
    wbase_other = np.concatenate([wbase[1:2], wbase[1:]])  # group 0 reads group 1's words
    for p, wb in [(pre_next, wbase), (pre, wbase_other)]:
        assert any(combine_compact(h, 0.5, n_pref, 5, wb, bits, p, partial) != combine_dense(h, 0.5, n_pref, 5, vbase, dense)
                   for h in range(n_pref[1]))
