"""The wide BC inputs of tests/test_gpu_bc_wide.py (wide_bc_inputs), proved on the CPU with the oracles alone.

BC's sigma is summed in fp64 at six steps of the device: the sigma[u] term, the warp accumulator and its xor tree
(bc_warp_sum), the stored segment partials of a vertex with more than SEG in-edges, bc_combine_kernel's accumulator,
bc_sigma_finish_kernel's store and the sigma[w] read of the delta term.  On the suite's older inputs every sigma is
below 2^24 or a power of two, so fp32 would hold every one of those values exactly.  Here a numpy model of the device's
sums (lanes strided over 32, the xor tree, SEG-edge segments combined in segment order) is run unnarrowed and with one
step narrowed to fp32 at a time:
  * unnarrowed it equals the oracle on every new input (sigma bit for bit; delta bit for bit on the lattice, at rtol
    1e-10 on the layered DAG), as the device must;
  * every narrowed variant fails that check on every new input from its root or corner (from the layered DAG's
    interior source all but the two hub-partial steps);
  * every narrowed variant passes it on the older inputs (RMAT-14/16 at the suite's sources, both forests, the small
    fixtures): the gap the new inputs close.
The oracles themselves are pinned here too: sigma of the layered DAG equals exact Python-integer path counts, and the
lattice's sigma and delta equal an independent recurrence over its anti-diagonals in both term orders.  Every case
asserts its own strength: how many sigma are >= 2^25 and not fp32 values, every hub segment partial >= 2^25, the hub
degrees at the segment boundaries, and sigma < 2^53 on the layered DAG."""
import functools

import numpy as np
import pytest

import bc_oracle as B
import bc_weighted_oracle as BW
from graphs import ALL_SMALL, in_degrees, rmat
from wide_bc_inputs import IN_HUB_BIG, IN_HUB_DEGREES, SEG, WIDE, lattice, layered, rn32, wide_count

STEPS = ("sigma_term", "warp_acc", "partial", "combine", "sigma_store", "delta_sigma_read")
INF = BW.INF


def f32(x):
    with np.errstate(over="ignore"):
        return rn32(x)


class Graph:
    """A CSC (with weights or not) and its push CSR (out-edges by ascending destination), as the device holds them."""

    def __init__(self, row_end, src, weight=None):
        nv = len(row_end)
        self.nv, self.src, self.weight = nv, np.asarray(src, np.int64), weight
        self.in_end = np.asarray(row_end, np.int64)
        self.in_beg = np.concatenate([[0], self.in_end[:-1]])
        self.dst = np.repeat(np.arange(nv), in_degrees(row_end))
        order = np.argsort(self.src, kind="stable")  # the CSC is by destination: out-lists come out ascending
        self.out_dst = self.dst[order]
        self.out_w = None if weight is None else np.asarray(weight, np.int64)[order]
        self.out_end = np.cumsum(np.bincount(self.src, minlength=nv))
        self.out_beg = np.concatenate([[0], self.out_end[:-1]])


def edges_of(beg, end, V):
    """The edges of the vertices V, concatenated: (edge index, index into V, position in the vertex's list)."""
    lens = end[V] - beg[V]
    owner = np.repeat(np.arange(len(V)), lens)
    pos = np.arange(int(lens.sum())) - np.repeat(np.cumsum(lens) - lens, lens)
    return beg[V][owner] + pos, owner, pos


def device_sum(term, owner, pos, n, narrow=(), hubs=None):
    """The device's sum of every vertex's terms (owner, pos: vertex and position in its list): lane = pos % 32 adds its
    terms in list order within a SEG-edge segment, the xor tree, then the segments' partials in segment order.
    `narrow` holds the steps rounded to fp32.  hubs: if a list, (index, partials) of every vertex with several segments
    is appended."""
    nseg = np.zeros(n, np.int64)
    np.maximum.at(nseg, owner, pos // SEG + 1)
    seg_base = np.cumsum(nseg) - nseg
    seg = seg_base[owner] + pos // SEG
    acc = np.zeros((int(nseg.sum()), 32))
    rnd = (pos % SEG) // 32
    order = np.argsort(rnd, kind="stable")
    cuts = np.searchsorted(rnd[order], np.arange(int(rnd.max()) + 2 if len(rnd) else 1))
    for r in range(len(cuts) - 1):
        e = order[cuts[r]:cuts[r + 1]]
        s, ln = seg[e], pos[e] % 32
        acc[s, ln] = acc[s, ln] + term[e]
        if "warp_acc" in narrow:
            acc[s, ln] = f32(acc[s, ln])
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, lanes ^ o]
        if "warp_acc" in narrow:
            acc = f32(acc)
    part = acc[:, 0]
    out = np.zeros(n)
    single = nseg == 1
    out[single] = part[seg_base[single]]
    if "partial" in narrow:
        part = f32(part)
    for v in np.nonzero(nseg > 1)[0]:
        p = part[seg_base[v]:seg_base[v] + nseg[v]]
        s = 0.0
        for x in p:
            s = f32(s + x) if "combine" in narrow else s + x
        out[v] = s
        if hubs is not None:
            hubs.append((v, p.copy()))
    return out


def model(g, key, s, narrow=(), delta=True, hubs=None):
    """sigma (and delta) of source s under the device's summation order; key = the oracle's lev (unweighted) or D."""
    weighted = g.weight is not None
    reached = key != INF if weighted else key < g.nv
    ids = np.nonzero(reached)[0]
    ids = ids[np.argsort(key[ids], kind="stable")]
    cut = np.concatenate([[0], np.nonzero(np.diff(key[ids]))[0] + 1, [len(ids)]])
    classes = [ids[cut[k]:cut[k + 1]] for k in range(len(cut) - 1)]
    kk = key.astype(np.int64)
    sigma = np.zeros(g.nv)
    sigma[s] = 1.0
    for V in classes[1:]:
        e, owner, pos = edges_of(g.in_beg, g.in_end, V)
        u = g.src[e]
        on = (reached[u] & (kk[u] + g.weight[e] == kk[V][owner])) if weighted else kk[u] == kk[V][owner] - 1
        t = np.where(on, f32(sigma[u]) if "sigma_term" in narrow else sigma[u], 0.0)
        cut_hubs = []
        out = device_sum(t, owner, pos, len(V), narrow, cut_hubs)
        if hubs is not None:
            hubs += [(int(V[j]), p) for j, p in cut_hubs]
        sigma[V] = f32(out) if "sigma_store" in narrow else out
    if not delta:
        return sigma, None
    dl = np.zeros(g.nv)
    for V in classes[-2::-1]:
        e, owner, pos = edges_of(g.out_beg, g.out_end, V)
        w = g.out_dst[e]
        on = (reached[w] & (kk[V][owner] + g.out_w[e] == kk[w])) if weighted else kk[w] == kk[V][owner] + 1
        sw = f32(sigma[w]) if "delta_sigma_read" in narrow else sigma[w]
        with np.errstate(divide="ignore", invalid="ignore"):
            t = np.where(on, (1.0 + dl[w]) / sw, 0.0)
        dl[V] = sigma[V] * device_sum(t, owner, pos, len(V))
    return sigma, dl


def oracle(g, s):
    if g.weight is None:
        lev, sigma, delta = B.source_state(g.in_end.astype(np.uint64), g.src, s)
    else:
        lev, sigma, delta = BW.source_state(g.in_end.astype(np.uint64), g.src, g.weight, s)
    return lev, sigma, delta


def holds(sigma, delta, ref_sigma, ref_delta, exact_delta):
    """The device's check: sigma bit for bit, delta bit for bit or at rtol 1e-10 with exact zeros."""
    if not np.array_equal(sigma, ref_sigma):
        return False
    if delta is None:
        return True
    if exact_delta:
        return np.array_equal(delta, ref_delta)
    return bool(np.array_equal(delta == 0, ref_delta == 0) and np.allclose(delta, ref_delta, rtol=1e-10, atol=0))


def variants_hold(g, s, exact_delta):
    """{step or "device": does the model with that step narrowed pass the device's check against the oracle}."""
    key, ref_sigma, ref_delta = oracle(g, s)
    out = {}
    for step in ("device",) + STEPS:
        narrow = () if step == "device" else (step,)
        sigma, delta = model(g, key, s, narrow, delta=step in ("device", "delta_sigma_read"))
        out[step] = holds(sigma, delta, ref_sigma, ref_delta, exact_delta)
    return out


# ---- the new inputs --------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def family(name, weighted):
    f = layered(weighted) if name == "layered" else lattice(weighted)
    return f, Graph(f["row_end"], f["src"], f["weight"])


NEW = [(name, weighted, which) for name in ("layered", "lattice") for weighted in (False, True) for which in ("root", "interior")]
MIN_WIDE = {("layered", "root"): 5000, ("layered", "interior"): 1500, ("lattice", "root"): 240000, ("lattice", "interior"): 190000}


@pytest.mark.parametrize("name,weighted,which", NEW)
def test_narrowed_models_fail_the_wide_inputs(name, weighted, which):
    f, g = family(name, weighted)
    s = f["sources"][which]
    key, ref_sigma, _ = oracle(g, s)
    assert wide_count(ref_sigma) >= MIN_WIDE[name, which], wide_count(ref_sigma)
    if name == "layered":
        assert ref_sigma.max() < 2.0 ** 53
    else:
        assert np.isfinite(ref_sigma).all()
    held = variants_hold(g, s, exact_delta=name == "lattice")
    assert held["device"], "the device model differs from the oracle"
    # from the layered DAG's interior source the hubs sit at sigma 2^23 to 2^26: only the root's hubs pin the partials
    must_fail = [k for k in STEPS if not (name == "layered" and which == "interior" and k in ("partial", "combine"))]
    assert not any(held[k] for k in must_fail), "narrowed steps the input cannot tell apart: %s" % [k for k in must_fail if held[k]]


@pytest.mark.parametrize("weighted", [False, True])
def test_layered_hubs_have_wide_partials_in_every_segment(weighted):
    f, g = family("layered", weighted)
    s = f["sources"]["root"]
    deg = in_degrees(f["row_end"])
    assert list(deg[f["in_hubs"]]) == list(IN_HUB_DEGREES) + [IN_HUB_BIG]
    assert np.bincount(g.src, minlength=g.nv)[f["out_hub"]] > SEG
    key, ref_sigma, _ = oracle(g, s)
    hubs = []
    sigma, _ = model(g, key, s, delta=False, hubs=hubs)
    assert np.array_equal(sigma, ref_sigma)
    seen = {int(v) for v, _ in hubs}
    assert seen >= set(int(h) for h in f["in_hubs"][1:]), "a cut hub was not summed in segments"
    for v, p in hubs:
        assert len(p) == -(-int(deg[v]) // SEG)
        assert np.all(p >= WIDE) and np.all(rn32(p) != p), "hub %d partials %s" % (v, np.log2(p))
    assert np.all(ref_sigma[f["in_hubs"]] >= WIDE)
    # the unsplit hub of exactly SEG edges is summed whole: wide too
    assert ref_sigma[f["in_hubs"][0]] >= WIDE and rn32(ref_sigma[f["in_hubs"][0]]) != ref_sigma[f["in_hubs"][0]]


@pytest.mark.parametrize("weighted", [False, True])
def test_layered_sigma_is_the_exact_path_count(weighted):
    f, g = family("layered", weighted)
    for which in ("root", "interior"):
        s = f["sources"][which]
        key, ref_sigma, _ = oracle(g, s)
        kk = key.astype(np.int64)
        reached = (key != INF) if weighted else (key < g.nv)
        exact = {int(s): 1}
        for v in np.nonzero(reached)[0][np.argsort(kk[reached], kind="stable")]:
            if v == s:
                continue
            u = g.src[g.in_beg[v]:g.in_end[v]]
            on = reached[u] & ((kk[u] + g.weight[g.in_beg[v]:g.in_end[v]] == kk[v]) if weighted else (kk[u] == kk[v] - 1))
            exact[int(v)] = sum(exact[int(x)] for x in u[on])
        assert max(exact.values()) < 2 ** 53
        got = {int(v): int(ref_sigma[v]) for v in np.nonzero(ref_sigma)[0]}
        assert got == {v: c for v, c in exact.items() if c}
        assert all(float(c) == ref_sigma[v] for v, c in exact.items())


def lattice_recurrence(n, a, b, swap):
    """sigma and delta of the lattice from (a, b) over its anti-diagonals, with the two terms of every sum in either
    order (missing terms are 0)."""
    S = np.zeros((n + 1, n + 1))
    D = np.zeros((n + 1, n + 1))
    T = np.zeros((n + 1, n + 1))
    m, k = n - a, n - b
    diag = [(np.arange(max(0, t - k + 1), min(t, m - 1) + 1)) for t in range(m + k - 1)]
    S[a, b] = 1.0
    with np.errstate(over="ignore"):
        for t in range(1, m + k - 1):
            i = a + diag[t]
            j = b + t - diag[t]
            up = np.where(i > a, S[i - 1, j], 0.0)
            left = np.where(j > b, S[i, j - 1], 0.0)
            S[i, j] = left + up if swap else up + left
        for t in range(m + k - 2, -1, -1):
            i = a + diag[t]
            j = b + t - diag[t]
            right, down = T[i, j + 1], T[i + 1, j]  # beyond the lattice: 0
            D[i, j] = S[i, j] * (down + right if swap else right + down)
            T[i, j] = (1.0 + D[i, j]) / S[i, j]
    return S[:n, :n].ravel(), D[:n, :n].ravel()


@pytest.mark.parametrize("weighted", [False, True])
def test_lattice_oracle_is_the_recurrence(weighted):
    f, g = family("lattice", weighted)
    n = f["n"]
    for which in ("root", "interior"):
        s = f["sources"][which]
        _, ref_sigma, ref_delta = oracle(g, s)
        for swap in (False, True):
            S, D = lattice_recurrence(n, s // n, s % n, swap)
            assert np.array_equal(S, ref_sigma) and np.array_equal(D, ref_delta)
        assert ref_sigma.max() > 2.0 ** 880 and np.isfinite(ref_delta).all()


@pytest.mark.parametrize("weighted", [False, True])
def test_lattice_hubs_hold_their_lattice_edges_at_the_chosen_positions(weighted):
    f, g = family("lattice", weighted)
    n = f["n"]
    deg_in, deg_out = in_degrees(f["row_end"]), np.bincount(g.src, minlength=g.nv)
    assert sorted(deg_in[f["in_hubs"]]) == sorted(deg_out[f["out_hubs"]]) == [SEG, SEG + 1, 3 * SEG + 1, 3 * SEG + 1]
    key, _, _ = oracle(g, f["sources"]["root"])
    kk = key.astype(np.int64)
    segs = set()
    for v, (q1, q2) in zip(f["in_hubs"], f["in_pos"]):
        e = np.arange(g.in_beg[v], g.in_end[v])
        u = g.src[e]
        on = (kk[u] + g.weight[e] == kk[v]) if weighted else kk[u] == kk[v] - 1
        assert list(np.nonzero(on)[0]) == [q1, q2] and list(u[[q1, q2]]) == [v - n, v - 1]
        segs |= {(-(-len(e) // SEG), q1 // SEG), (-(-len(e) // SEG), q2 // SEG)}
    for x, (q1, q2) in zip(f["out_hubs"], f["out_pos"]):
        e = np.arange(g.out_beg[x], g.out_end[x])
        w = g.out_dst[e]
        on = (kk[x] + g.out_w[e] == kk[w]) if weighted else kk[w] == kk[x] + 1
        assert list(np.nonzero(on)[0]) == [q1, q2] and list(w[[q1, q2]]) == [x + 1, x + n]
        segs |= {(-(-len(e) // SEG), q1 // SEG), (-(-len(e) // SEG), q2 // SEG)}
    # lattice edges in the first, a middle and the last segment of the 3 SEG + 1 lists, and in the lone last edge
    assert {(4, 0), (4, 1), (4, 2), (4, 3), (2, 0), (2, 1)} <= segs


# ---- the older inputs ------------------------------------------------------------------------------------------------
OLD = ["rmat14", "rmat16", "forest", "weighted_forest"] + ["small_" + n for n in sorted(ALL_SMALL)]


def old_case(name):
    """(row_end, src, weight, sources, delta bit for bit) of an older input at the suite's sources (a few per small
    fixture)."""
    if name.startswith("rmat"):
        scale = int(name[4:])
        row_end, src = rmat(scale)
        return row_end, src, None, np.random.default_rng(scale).choice(len(row_end), 8, replace=False), False
    if name.endswith("forest"):
        f = (BW if name == "weighted_forest" else B).forest()
        return f["row_end"], f["src"], f.get("weight"), f["roots"][:6], True
    row_end, src = ALL_SMALL[name[6:]]()
    nv = len(row_end)
    return row_end, src, None, np.unique(np.concatenate([[0, nv - 1], np.random.default_rng(1).choice(nv, 4, replace=False)])), False


@pytest.mark.parametrize("name", OLD)
def test_narrowed_models_pass_the_older_inputs(name):
    row_end, src, weight, sources, exact_delta = old_case(name)
    g = Graph(row_end, src, weight)
    for s in sources:
        held = variants_hold(g, int(s), exact_delta)
        assert all(held.values()), "%s source %d: %s" % (name, s, held)
