"""Exact betweenness-centrality inputs whose path counts outgrow fp32 (test infrastructure only).

The suite's other BC inputs keep every sigma below 2^24 (RMAT, the small fixtures) or make it a power of two (the
forests), where fp32 holds every term and every partial sum exactly: a sweep whose fp64 sigma had been narrowed to fp32
would still match the oracle bit for bit.  The two families here do not allow that.

  layered(): a layered DAG.  A source, then `depth` layers of `width` vertices; every vertex draws `parents` distinct
    parents from the previous layer with multiplicities 1 to 5, so sigma grows by about 2^7 per layer and reaches 2^45.
    Every sigma is an integer below 2^53, so every summation order gives the same fp64 value: sigma is bit for bit,
    delta and the scores are compared at rtol 1e-10.  In-degree hubs of exactly SEG, SEG + 1, 2 SEG + 1, 3 SEG + 1 and
    IN_HUB_BIG edges sit one layer past sigma ~ 2^30, with same-level and backward decoys interleaved by id, matching
    edges in every segment; an out-degree hub sends more than SEG edges to the next layer.

  lattice(): the directed n x n lattice, (i, j) -> (i + 1, j) and (i, j) -> (i, j + 1), id = i * n + j.  From (a, b),
    sigma(i, j) = C(i - a + j - b, i - a), far past 2^53 (2^992.7 at the far corner of n = 500; n = 520 overflows).
    Every sigma sum and every delta sum has at most two non-zero terms, and x + 0, a + b = b + a are exact in IEEE
    arithmetic, so each value is one rounding of the same inputs in every lane order, segment split and rank split:
    lev, sigma, delta and the scores equal the oracle bit for bit.  Decoy in- and out-edges make a few vertices cross
    SEG, SEG + 1 and 3 SEG + 1 edges with their two lattice edges in chosen segments.

Both come unweighted (LUXB_BC) and weighted (LUXB_BC_WEIGHTED).  Weighted layered: every tight edge has weight
TIGHT_W; decoys also include heavier parallel copies of tight edges.  Weighted lattice: weight 2 on (i + 1, j), 1 on
(i, j + 1), so every lattice edge is tight, D(i, j) = 2 i + j and sigma / delta equal the unweighted ones bit for bit;
its decoys are non-tight (heavier parallel copies, or D[u] + w > D[v]).  A decoy never matches the level or tight
filter and never shortens a path, from any of the family's sources."""
import numpy as np

import oracle as O
import bc_weighted_oracle as BW

SEG = 4096                      # kBcSegment of bc.cuh: edges per hub segment
IN_HUB_DEGREES = (SEG, SEG + 1, 2 * SEG + 1, 3 * SEG + 1)
IN_HUB_BIG = 30000
TIGHT_W = 7                     # the weight of every tight edge of the weighted layered DAG
LATTICE_N = 500                 # 520 already overflows: 45 sigma are inf
WIDE = 2.0 ** 25


def rn32(x):
    with np.errstate(over="ignore"):
        return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def wide_count(sigma):
    """The sigma >= 2^25 that fp32 cannot hold."""
    s = np.asarray(sigma)
    return int(np.count_nonzero((s >= WIDE) & (rn32(s) != s)))


def _spread(rng, total, k):
    """`total` edges over k groups, every group >= 1 (k <= total)."""
    return 1 + rng.multinomial(total - k, np.full(k, 1.0 / k)) if k else np.zeros(0, np.int64)


def _finish(nv, es, ed, ew, weighted, **info):
    es, ed = np.concatenate(es).astype(np.int64), np.concatenate(ed).astype(np.int64)
    if weighted:
        row_end, src, weight = BW.edges_to_csc(nv, es, ed, np.concatenate(ew))
    else:
        (row_end, src), weight = O.edges_to_csc(nv, es, ed), None
    return dict(row_end=row_end, src=src, weight=weight, **info)


# ---- (A) the layered DAG ----------------------------------------------------------------------------------------------
def layered(weighted=False, seed=1, width=2048, depth=7, parents=48, hub_layer=6):
    """dict(row_end, src, weight (None unweighted), sources = {root, interior, multi}, in_hubs (ids, the degrees of
    IN_HUB_DEGREES then IN_HUB_BIG), out_hub, layer (of every id; -1: none))."""
    rng = np.random.default_rng(seed)
    n_hub = len(IN_HUB_DEGREES) + 1
    nv = 1 + width * depth + n_hub
    perm = rng.permutation(nv)           # logical vertex -> id: layers and hubs interleave in id order
    layer = np.concatenate([[0], np.repeat(np.arange(1, depth + 1), width), np.full(n_hub, hub_layer)])
    members = [np.array([0])] + [1 + width * (k - 1) + np.arange(width) for k in range(1, depth + 1)]
    es, ed, ew = [], [], []

    def add(s, d, w):
        es.append(perm[s]); ed.append(perm[d]); ew.append(np.broadcast_to(np.asarray(w, np.int64), np.shape(s)))

    for k in range(1, depth + 1):
        prev = members[k - 1]
        for v in members[k]:
            p = rng.choice(prev, min(parents, len(prev)), replace=False)
            m = rng.integers(1, 6, len(p))
            add(np.repeat(p, m), np.full(int(m.sum()), v), TIGHT_W)
        # a few decoys per vertex: from its own layer or a deeper one (never on the level filter, never shorter)
        nd = rng.integers(0, 4, width)
        v = np.repeat(members[k], nd)
        u = 1 + rng.integers(width * (k - 1), width * depth, len(v))
        add(u, v, rng.integers(1, 256, len(v)))
    # the out-degree hub: one vertex of the layer before the hubs becomes a parent of its whole next layer
    out_hub = int(members[hub_layer - 1][0])
    m = rng.integers(2, 5, width)
    add(np.full(int(m.sum()), out_hub), np.repeat(members[hub_layer], m), TIGHT_W)
    # the in-degree hubs: parents from the layer before, decoys from their own layer and deeper, sorted by id
    par_pool, dec_pool = members[hub_layer - 1], np.concatenate(members[hub_layer:])
    hubs = 1 + width * depth + np.arange(n_hub)
    for h, total in zip(hubs, IN_HUB_DEGREES + (IN_HUB_BIG,)):
        nseg = -(-total // SEG)
        p = rng.choice(par_pool, 12 * nseg, replace=False)
        pm = rng.integers(1, 6, len(p))
        heavy = rng.integers(0, 3, len(p)) if weighted else np.zeros(len(p), np.int64)
        last = np.argmax(perm[p])  # the highest id is a parent: the lone last edge of a cut hub is a tight one
        heavy[last] = 0
        d = rng.choice(dec_pool[perm[dec_pool] < perm[p[last]]], 64 * nseg, replace=False)
        dm = _spread(rng, total - int(pm.sum() + heavy.sum()), len(d))
        for x, mm, hh in zip(p, pm, heavy):  # a heavier copy of a tight edge is a decoy too
            add(np.full(mm + hh, x), np.full(mm + hh, h), np.concatenate([np.full(mm, TIGHT_W), TIGHT_W + rng.integers(1, 9, hh)]))
        add(np.repeat(d, dm), np.full(int(dm.sum()), h), rng.integers(1, 256, int(dm.sum())))
    interior = int(members[1][5])
    g = _finish(nv, es, ed, ew, weighted, in_hubs=perm[hubs].astype(np.uint32), out_hub=int(perm[out_hub]),
                sources=dict(root=int(perm[0]), interior=int(perm[interior]),
                             multi=np.array([perm[0], perm[interior], perm[members[2][9]]], np.uint32)))
    lay = np.full(nv, -1, np.int64)
    lay[perm] = layer
    g["layer"] = lay
    return g


# ---- (B) the directed lattice -----------------------------------------------------------------------------------------
LATTICE_SOURCES = ((0, 0), (60, 45), (95, 20))
# in-edge hubs: (i, j), total in-degree, positions of the edges from (i - 1, j) and (i, j - 1) in its CSC list
LATTICE_IN_HUBS = (((250, 250), SEG, 0, SEG - 1), ((300, 220), SEG + 1, 2000, SEG), ((220, 330), 3 * SEG + 1, SEG + 1234, 3 * SEG),
                   ((330, 260), 3 * SEG + 1, 0, 2 * SEG + 5))
# out-edge hubs: (i, j), total out-degree, positions of the edges to (i, j + 1) and (i + 1, j) in its out-list
LATTICE_OUT_HUBS = (((260, 240), SEG, 0, SEG - 1), ((310, 180), SEG + 1, 1500, SEG), ((200, 300), 3 * SEG + 1, 5, 2 * SEG + 77),
                    ((280, 290), 3 * SEG + 1, SEG + 9, 3 * SEG))


def lattice_corner(n=LATTICE_N):
    """The least vertex every lattice source reaches: decoys only touch vertices at or past it."""
    return max(a for a, _ in LATTICE_SOURCES), max(b for _, b in LATTICE_SOURCES)


def lattice(weighted=False, n=LATTICE_N, seed=2):
    """dict(row_end, src, weight (None unweighted), n, sources = {root, interior, multi} (ids), in_hubs / out_hubs (ids),
    in_pos / out_pos (the lattice edges' positions in each hub's list))."""
    rng = np.random.default_rng(seed)
    nv = n * n
    ids = np.arange(nv).reshape(n, n)
    lev0 = (ids // n) + (ids % n)
    d0 = 2 * (ids // n) + (ids % n)
    lev0, d0 = lev0.ravel(), d0.ravel()
    es = [ids[:-1, :].ravel(), ids[:, :-1].ravel()]
    ed = [ids[1:, :].ravel(), ids[:, 1:].ravel()]
    ew = [np.full(n * (n - 1), 2), np.full(n * (n - 1), 1)]
    ci, cj = lattice_corner(n)
    past = ((ids // n) >= ci) & ((ids % n) >= cj)
    past = past.ravel()

    def decoy_w(u, v):
        """A non-tight weight for u -> v (D[u] + w > D[v] from every source)."""
        gap = d0[v] - d0[u]
        return np.where(gap >= 0, gap + 1 + rng.integers(0, 40, len(u)), rng.integers(1, 256, len(u)))

    def fill(lo, hi, count, ok):
        """`count` decoy edge ends among the ids [lo, hi) for which ok(ids) holds, ascending, a few distinct ids."""
        if count == 0:
            return np.zeros(0, np.int64)
        cand = np.arange(lo, hi)
        cand = cand[ok(cand)]
        k = min(len(cand), max(1, count // 40), count)
        assert k > 0, "no decoy ids in [%d, %d)" % (lo, hi)
        return np.repeat(np.sort(rng.choice(cand, k, replace=False)), _spread(rng, count, k))

    heavy = 3 if weighted else 0
    in_hubs, in_pos = [], []
    for (i, j), total, q1, q2 in LATTICE_IN_HUBS:
        v = i * n + j
        p1, p2 = v - n, v - 1
        assert past[v] and q1 + 1 + 2 * heavy <= q2 < total
        ok = lambda u: lev0[u] >= lev0[v]  # noqa: E731  same level or deeper: never on the level filter
        u = np.concatenate([fill(0, p1, q1, ok), np.full(1 + heavy, p1), fill(p1 + 1, p2, q2 - q1 - 1 - 2 * heavy, ok),
                            np.full(heavy + 1, p2), fill(p2 + 1, nv, total - q2 - 1, ok)])
        w = decoy_w(u, np.full(len(u), v))
        w[q1] = 2
        w[q1 + 1:q1 + 1 + heavy] = 2 + rng.integers(1, 9, heavy)
        w[q2 - heavy:q2] = 1 + rng.integers(1, 9, heavy)
        w[q2] = 1
        assert len(u) == total
        es.append(u); ed.append(np.full(total, v)); ew.append(w)
        in_hubs.append(v); in_pos.append((q1, q2))
    out_hubs, out_pos = [], []
    for (i, j), total, q1, q2 in LATTICE_OUT_HUBS:
        x = i * n + j
        c1, c2 = x + 1, x + n
        assert q1 + 1 + 2 * heavy <= q2 < total
        ok = lambda y: (lev0[y] <= lev0[x]) & past[y]  # noqa: E731  reached from every source, never deeper than x
        y = np.concatenate([fill(0, c1, q1, ok), np.full(1 + heavy, c1), fill(c1 + 1, c2, q2 - q1 - 1 - 2 * heavy, ok),
                            np.full(heavy + 1, c2), fill(c2 + 1, nv, total - q2 - 1, ok)])
        w = decoy_w(np.full(len(y), x), y)
        w[q1] = 1
        w[q1 + 1:q1 + 1 + heavy] = 1 + rng.integers(1, 9, heavy)
        w[q2 - heavy:q2] = 2 + rng.integers(1, 9, heavy)
        w[q2] = 2
        assert len(y) == total
        es.append(np.full(total, x)); ed.append(y); ew.append(w)
        out_hubs.append(x); out_pos.append((q1, q2))
    # the hubs' own lattice edges are in the edge lists twice now: drop the first copies
    drop_in = np.isin(ed[0], in_hubs) | np.isin(es[0], out_hubs)  # (i - 1, j) -> (i, j) and (i, j) -> (i + 1, j)
    drop_right = np.isin(ed[1], in_hubs) | np.isin(es[1], out_hubs)
    es[0], ed[0], ew[0] = es[0][~drop_in], ed[0][~drop_in], ew[0][~drop_in]
    es[1], ed[1], ew[1] = es[1][~drop_right], ed[1][~drop_right], ew[1][~drop_right]
    src_ids = [a * n + b for a, b in LATTICE_SOURCES]
    return _finish(nv, es, ed, ew, weighted, n=n, in_hubs=np.array(in_hubs, np.uint32), out_hubs=np.array(out_hubs, np.uint32),
                   in_pos=in_pos, out_pos=out_pos,
                   sources=dict(root=src_ids[0], interior=src_ids[1], multi=np.array(src_ids, np.uint32)))
