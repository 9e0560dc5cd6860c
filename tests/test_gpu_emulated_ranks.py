"""GPU: the multi-rank paths on one device.  World = 2, 3 or 4 ranks (64 where noted) run as host threads of one
process on device 0, exchanging through the in-process NCCL stand-in (tests/fake_nccl.c, pinned on the CPU by
tests/test_fake_nccl.py; tests/emu_ranks.py runs each case in its own subprocess).  Every rank's result is compared with
the oracles, bit for bit wherever the inputs make it exact; each case first asserts the property it is named after.

  * partitions: bounds() equals O.partition on every rank for from_csc, from_rmat (plain, balanced, weighted),
    from_bipartite (plain, balanced) and from_file; the local_csc() slices rebuild the whole CSC, with the generators'
    edge weights (row_left / col_left offsets); out_degree() is the global out-degree (the degree all-reduce);
    balanced=True keeps the reference split in bounds() and works on a contiguous cover; every opened handle runs its
    app against the oracle (PageRank exact steps, CF, weighted SSSP with the trace of label_run(P=world));
  * PageRank through the NCCL exchange (grouped broadcasts of the packed hot / cold ranges): one exact step from
    set_values, bit-equal to O.pagerank_iter, on the plain seg stream, the forced panel split, the merge path,
    zero-copy edges and the balanced split (the panel, merge and zero-copy paths asserted through the panel edges
    under forced-split settings and the edges' memory type), at RMAT-16 and on the small fixtures the partitioner cuts into `world`
    parts; set_local_values / local_values round trips; 6 iterations against O.pagerank at 1e-6;
  * CC / SSSP / weighted SSSP stepped iteration by iteration: labels against label_pull^k, the active count, EVERY
    rank's frontier representation against the oracle's ftype[k, rank], the trace against label_run(P=world); the
    designed cases of test_frontier_cases_model.py and the fixtures, a graph on which a partition pushes from a
    bitmap frontier, cases where a partition's queue overflows and is promoted; check() summed over the ranks equals
    the oracle's count on perturbed labels, and the run from them (set_values restart) reaches a state check() accepts;
  * collaborative filtering: one exact step (cf_exact_step), the items' factors 10-19 bit for bit, the rest at 2e-6;
  * BC and weighted BC: the exact forests bit for bit (lev, sigma, delta, scores); RMAT-14 lev and sigma bit for bit,
    delta and scores at rtol 1e-10; a last partition without edges;
  * TC: t and T bit for bit against the oracle on every rank (and every rank's local_values()), on RMAT-14 from the
    device generator, RMAT-16 balanced, K_300 stored both ways and an edge-free last partition;
  * graphs the reference partitioner cannot cut into `world` parts (edge-free and vertex-free partitions, and the
    64-rank pass): every app, weighted BC included, runs, and its result equals the one-rank oracle;
  * exchange=P2P without a peer import takes the NCCL path and gives the EXCHANGE_NCCL results.
Not covered here: the P2P exchange itself (the flag barrier, pack_push / chunk_pull, frontier_push, CF's peer stores),
the stream ordering of real asynchronous collectives, and NCCL's float summation order (the stand-in sums in rank order;
only exact inputs or tolerances are asserted on float all-reduces).  LUXB_SKIP_HEAVY=1 skips the large forests."""
import ctypes as C
import functools
import os
import shutil
import tempfile

import numpy as np
import pytest

import lux_b200 as L
import oracle as O
import bc_oracle as B
import bc_weighted_oracle as BW
import tc_oracle as T
import weighted_oracle as W
from emu_ranks import emulate, run_ranks
from graphs import ALL_SMALL, exact_pr_inputs, in_degrees, rmat, symmetrize
from mgpu_bc_worker import edge_free_case
from test_gpu_exact import cf_exact_step, exact_steps
from test_frontier_cases_model import CASE_RUNS, CC, FIXTURE_RUNS, SSSP, WSSSP, build_run, case_run_id, jacobi, reference

pytestmark = pytest.mark.gpu
heavy = pytest.mark.skipif(os.environ.get("LUXB_SKIP_HEAVY") == "1", reason="LUXB_SKIP_HEAVY=1")
WORLDS = [2, 3, 4]
LAPP = {CC: L.APP_CC, SSSP: L.APP_SSSP, WSSSP: L.APP_SSSP_WEIGHTED}
OAPP = {CC: O.APP_CC, SSSP: O.APP_SSSP}
PANEL = dict(LUXB_SB=1, LUXB_SB_BS=64, LUXB_SB_MIN_INDEG=4)


def first_diff(got, want, what):
    """Bit-for-bit comparison (floats by their bits) naming the first differing index."""
    g, w = np.asarray(got), np.asarray(want)
    assert g.shape == w.shape, "%s: shape %s, want %s" % (what, g.shape, w.shape)
    if g.dtype.kind == "f":
        bits = np.dtype("u%d" % g.dtype.itemsize)
        g, w = g.view(bits), w.astype(g.dtype).view(bits)
    bad = np.nonzero(g.reshape(-1) != w.reshape(-1))[0]
    assert bad.size == 0, "%s: %d values differ, first at flat index %d: got %r, want %r" % (
        what, bad.size, bad[0], np.asarray(got).reshape(-1)[bad[0]], np.asarray(want).reshape(-1)[bad[0]])


def close(got, want, what, rtol):
    bad = np.nonzero(~np.isclose(got, want, rtol=rtol, atol=0) | ((got == 0) != (want == 0)))[0]
    assert bad.size == 0, "%s: %d values off by more than rtol %g, first at %d: got %r, want %r" % (
        what, bad.size, rtol, bad[0], got[bad[0]], want[bad[0]])


def opened(uid, i, world, rank, row_end, src, w=None, **kw):
    g = L.LuxGraph.from_csc(row_end, src, w, rank=rank, nranks=world, device=0, **kw)
    g.comm_init(uid(i))
    g.init()
    return g


def parts(row_end, src, world):
    return int(O.partition(row_end, len(src), world)[0])


@functools.lru_cache(maxsize=None)
def graph(name):
    if name in ALL_SMALL:
        return ALL_SMALL[name]()
    if name.endswith("_sym"):
        return symmetrize(*rmat(int(name[4:-4]), ef=8))
    return rmat(int(name[4:]))


def bitmap_push_graph():
    """40 000 vertices: a 2 000-vertex chain from 0, 8 random in-edges into each of the top 4 000 vertices and 1 000
    out-edges from vertex 0 into the top range.  At P = 2 the top range is one partition, whose frontier after the first
    SSSP iteration is a bitmap (1 000 of about 5 500 vertices) that the next iteration pushes from."""
    nv, top, chain, fan = 40000, 4000, 2000, 1000
    rng = np.random.default_rng(1)
    lo = nv - top
    a = np.concatenate([np.arange(chain - 1), rng.integers(0, nv, 8 * top), np.zeros(fan, np.int64)])
    b = np.concatenate([np.arange(1, chain), np.repeat(np.arange(lo, nv), 8), lo + rng.choice(top, fan, replace=False)])
    row_end, src = O.edges_to_csc(nv, a, b)
    return row_end, src, np.random.default_rng(2).integers(1, 256, len(src)).astype(np.int32)


def oracle_run(app, row_end, src, w, start, P):
    if app == WSSSP:
        return W.label_run(row_end, src, w, P=P, start=start)
    return O.label_run(OAPP[app], row_end, src, P=P, start=start)


def label_check(app, row_end, src, w, lab):
    return W.label_check(row_end, src, w, lab) if app == WSSSP else O.label_check(OAPP[app], row_end, src, lab)


# ---- cases (run inside the emulating subprocess) ---------------------------------------------------------------------
def case_partitions(world):
    """Every opener: the partition table, the local slices (with the generators' edge weights, whose keys carry the
    destination minus row_left), the degree all-reduce, and one run of the opened app against the oracle."""
    re16, src16 = graph("rmat16")
    w16 = W.rmat_weights(27, re16, src16)
    users, items, ratings = 4000, 200, 200000
    reb, srcb, wb = O.gen_bipartite_csc(users, items, ratings, 5)
    tmp = tempfile.mkdtemp(prefix="luxb_emu_")
    lux = os.path.join(tmp, "rmat12.lux")
    re12, src12 = graph("rmat12_ragged_nv")
    O.lux_write(lux, re12, src12)
    kw = lambda r: dict(rank=r, nranks=world, device=0)  # noqa: E731
    rmat = lambda r, **k: L.LuxGraph.from_rmat(16, 1 << 16, 16 << 16, 27, **kw(r), **k)  # noqa: E731
    # (name, opener, row_end, src, weights the slices must carry or None)
    openers = [("rmat16", lambda r: rmat(r), re16, src16, None),
               ("balanced rmat16", lambda r: rmat(r, balanced=True), re16, src16, None),
               ("weighted rmat16", lambda r: rmat(r, app=L.APP_SSSP_WEIGHTED, start=0), re16, src16, w16),
               ("csc rmat16", lambda r: L.LuxGraph.from_csc(re16, src16, **kw(r)), re16, src16, None),
               ("balanced csc", lambda r: L.LuxGraph.from_csc(re16, src16, balanced=True, **kw(r)), re16, src16, None),
               ("bipartite", lambda r: L.LuxGraph.from_bipartite(users, items, ratings, 5, **kw(r)), reb, srcb, wb),
               ("balanced bipartite", lambda r: L.LuxGraph.from_bipartite(users, items, ratings, 5, balanced=True, **kw(r)),
                reb, srcb, wb),
               ("file", lambda r: L.LuxGraph.from_file(lux, **kw(r)), re12, src12, None)]
    for name, _, row_end, src, _ in openers:
        assert parts(row_end, src, world) == world, "%s does not partition into %d" % (name, world)
    ref_sssp = W.label_run(re16, src16, w16, P=world, start=0)
    ref_cf = O.colfilter(reb, srcb, wb, 3)

    def body(rank, uid):
        got = []
        for i, (name, open_, row_end, src, weight) in enumerate(openers):
            cnt, rl, rr, cl, fl, fr = O.partition(row_end, len(src), world)
            what = "%s rank %d" % (name, rank)
            with open_(rank) as g:
                b = g.bounds()
                assert b["found"] == cnt, what
                for k, want in (("row_left", rl), ("row_right", rr), ("col_left", cl), ("fq_left", fl), ("fq_right", fr)):
                    first_diff(b[k], want, "%s %s" % (what, k))
                wb_ = g.work_bounds()
                if name.startswith("balanced"):
                    assert wb_["balanced"] and int(wb_["row_left"][0]) == 0 and int(wb_["row_right"][-1]) == len(row_end) - 1, what
                    assert all(int(wb_["row_right"][p]) + 1 == int(wb_["row_left"][p + 1]) for p in range(world - 1)), what
                    assert not np.array_equal(wb_["row_left"], rl), "%s: the balanced cuts are the reference cuts" % what
                else:
                    assert not wb_["balanced"] and np.array_equal(wb_["row_left"], rl), what
                lo, n = g.local_range()
                assert (lo, n) == (int(wb_["row_left"][rank]), int(wb_["row_right"][rank]) - int(wb_["row_left"][rank]) + 1), what
                slc = g.local_csc(weighted=weight is not None)
                g.comm_init(uid(i))
                g.init()
                if g.app == L.APP_PAGERANK:
                    first_diff(g.out_degree(), O.out_degree(len(row_end), src), what + " out_degree")
                    exact_steps(g, row_end, src, what)
                elif g.app == L.APP_COLFILTER:
                    g.set_values(O.cf_init(len(row_end)))
                    g.iterate(3)
                    close(g.values().reshape(-1), ref_cf.reshape(-1), what + " cf 3 iterations", 2e-6)
                else:
                    assert g.run_to_convergence() == ref_sssp["iters"], what
                    first_diff(g.values(), ref_sssp["labels"], what + " weighted sssp labels")
                    active, pull = g.trace()
                    first_diff(active, ref_sssp["active"], what + " trace active")
                    first_diff(pull, ref_sssp["pull"], what + " trace pull")
                got.append(slc)
        return got

    try:
        out = run_ranks(world, body)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    for i, (name, _, row_end, src, weight) in enumerate(openers):
        first_diff(np.concatenate([out[r][i][0] for r in range(world)]), row_end, name + ": concatenated local row_end")
        first_diff(np.concatenate([out[r][i][1] for r in range(world)]), src, name + ": concatenated local src")
        if weight is not None:
            first_diff(np.concatenate([out[r][i][2] for r in range(world)]), weight, name + ": concatenated local weights")


def edges_in_host_memory(g):
    """The handle's edge array is mapped host memory (cuPointerGetAttribute, in the rank's current context)."""
    cu = C.CDLL("libcuda.so.1")
    kind = C.c_uint(0)
    rc = cu.cuPointerGetAttribute(C.byref(kind), C.c_int(2), C.c_ulonglong(g.device_view().src))  # MEMORY_TYPE
    assert rc == 0, "cuPointerGetAttribute failed (%d)" % rc
    return kind.value == 1  # CU_MEMORYTYPE_HOST


def case_pagerank(world, names, zero_copy=False, balanced=False, exchange=L.EXCHANGE_NCCL, sweep="seg"):
    """sweep names the path the pull sweep must take on RMAT-16: "panel" (forced split, panel edges), "seg", or "merge"
    (both run with the forced-split settings in the environment, so that a sweep that fell back to the flagged stream
    would show panel edges)."""
    graphs = [n for n in names if parts(*graph(n), world) == world]
    assert graphs, "no graph partitions into %d" % world

    def body(rank, uid):
        for i, name in enumerate(graphs):
            row_end, src = graph(name)
            nv = len(row_end)
            what = "pagerank %s rank %d" % (name, rank)
            with opened(uid, i, world, rank, row_end, src, zero_copy=zero_copy, balanced=balanced, exchange=exchange) as g:
                if name == "rmat16" and sweep is not None:
                    pe = g.stats()["panel_edges"]
                    assert (pe > 0) == (sweep == "panel"), "%s: %d panel edges on the %s path" % (what, pe, sweep)
                if zero_copy:
                    assert edges_in_host_memory(g), what + ": the edges are not in mapped host memory"
                exact_steps(g, row_end, src, what, rounds=2)
                deg = O.out_degree(nv, src)
                lo, n = g.local_range()
                y = exact_pr_inputs(nv, max(int(in_degrees(row_end).max()), 1), salt=5)[0]
                g.set_local_values(y[lo:lo + n])
                first_diff(g.local_values(), y[lo:lo + n], what + " local_values after set_local_values")
                g.iterate(1)
                x = g.values()
                first_diff(x, O.pagerank_iter(row_end, src, deg, y), what + " one step from set_local_values")
                first_diff(g.local_values(), x[lo:lo + n], what + " local_values")
                g.set_values(O.pagerank_init(deg))
                g.iterate(6)
                ref = O.pagerank(row_end, src, 6)
                close(g.values(), ref, what + " 6 iterations", 1e-6)

    run_ranks(world, body)


def label_properties(plans):
    """What the oracle's runs at P = world show: a push from a partition's bitmap frontier, a push whose new frontier
    overflows the queue on some partitions only (promoted to a bitmap there)."""
    seen = set()
    for run, _, _, _, _, orc in plans:
        dense = orc["ftype"] == O.DENSE_BITMAP
        push = orc["pull"] == 0
        if any(push[k] and dense[k - 1].any() for k in range(1, len(push))):
            seen.add("bitmap push")
        if any(push[k] and dense[k].any() and not dense[k].all() for k in range(len(push))):
            seen.add("promotion on one partition")
    return seen


def label_plans(world, runs):
    """(run, row_end, src, w, one-rank reference, oracle at P = world) of every run whose graph the reference cuts into
    `world` parts."""
    plans = []
    for run in runs:
        name, app, start = run
        row_end, src, w, _ = build_run(name) if name != "bitmap_push" else (*bitmap_push_graph(), None)
        if parts(row_end, src, world) != world:
            continue
        ref = reference(app, row_end, src, w, start)
        orc = oracle_run(app, row_end, src, w, start, world)
        assert orc["iters"] == ref.iters and np.array_equal(orc["active"], ref.active), case_run_id(run)
        plans.append((run, row_end, src, w, ref, orc))
    assert plans, "no run partitions into %d" % world
    return plans


def restart_plan(app, row_end, src, w, ref):
    """Perturbed labels (CC: random; SSSP: the fixpoint plus 0..3, clipped to INF), the run from them and the oracle's
    check() count on them."""
    nv = len(row_end)
    rng = np.random.default_rng(17)
    if app == CC:
        lab0 = rng.integers(0, nv, nv).astype(np.uint32)
    else:
        inf = nv if app == SSSP else W.INF
        lab0 = np.minimum(ref.labels[-1].astype(np.int64) + rng.integers(0, 4, nv), inf).astype(np.uint32)
    return lab0, jacobi(app, row_end, src, w, lab0, nv), label_check(app, row_end, src, w, lab0)


def step_label_runs(world, plans, restart):
    """Every plan stepped on every rank, one iterate(1) at a time; with `restart`, then set_values of perturbed labels
    and the run from them."""
    restarts = [restart_plan(run[1], row_end, src, w, ref) if restart else None for run, row_end, src, w, ref, _ in plans]

    def body(rank, uid):
        checks = []
        for i, ((run, row_end, src, w, ref, orc), rs) in enumerate(zip(plans, restarts)):
            name, app, start = run
            what = "%s rank %d/%d" % (case_run_id(run), rank, world)
            with opened(uid, i, world, rank, row_end, src, w if app == WSSSP else None, app=LAPP[app], start=start) as g:
                for k in range(ref.iters):
                    act = g.iterate(1)
                    lab = g.values()
                    first_diff(lab, ref.labels[k + 1], "%s iteration %d labels" % (what, k))
                    assert act == ref.active[k], "%s iteration %d: active %d, want %d" % (what, k, act, ref.active[k])
                    ft = g.stats()["last_frontier_type"]
                    assert ft == orc["ftype"][k, rank], "%s iteration %d: frontier type %#x, want %#x" % (
                        what, k, ft, orc["ftype"][k, rank])
                active, pull = g.trace()
                first_diff(active, orc["active"], what + " trace active")
                first_diff(pull, orc["pull"], what + " trace pull")
                row = [g.check()]
                if rs is not None:
                    lab0, again, _ = rs
                    g.set_values(lab0)
                    row.append(g.check())
                    for k in range(again.iters):
                        act = g.iterate(1)
                        first_diff(g.values(), again.labels[k + 1], "%s restart iteration %d labels" % (what, k))
                        assert act == again.active[k], "%s restart iteration %d: active %d, want %d" % (what, k, act, again.active[k])
                    row.append(g.check())
                checks.append(row)
        return checks

    out = run_ranks(world, body)
    for i, ((run, row_end, src, w, ref, orc), rs) in enumerate(zip(plans, restarts)):
        rows = [out[r][i] for r in range(world)]
        assert sum(r[0] for r in rows) == 0, "%s: check() after convergence" % case_run_id(run)
        if rs is not None:
            assert sum(r[1] for r in rows) == rs[2], "%s: check() summed over ranks %d, oracle %d on perturbed labels" % (
                case_run_id(run), sum(r[1] for r in rows), rs[2])
            assert sum(r[2] for r in rows) == 0, "%s: check() after the restarted run" % case_run_id(run)


LABEL_GROUPS = {"cases": CASE_RUNS, "fixtures": FIXTURE_RUNS,
                "bitmap": [("bitmap_push", SSSP, 0), ("bitmap_push", WSSSP, 0), ("bitmap_push", CC, 0)]}


def case_labels(world, group, restart=False):
    plans = label_plans(world, LABEL_GROUPS[group])
    seen = label_properties(plans)
    if group == "cases":
        assert "promotion on one partition" in seen, seen
    if group == "bitmap" and world == 2:
        assert "bitmap push" in seen, seen
    step_label_runs(world, plans, restart)


def case_colfilter(world):
    cases = [(300, 40, 20000), (4000, 200, 200000)]

    def body(rank, uid):
        for i, (users, items, ratings) in enumerate(cases):
            row_end, src, w = O.gen_bipartite_csc(users, items, ratings, 5)
            with opened(uid, i, world, rank, row_end, src, w, app=L.APP_COLFILTER) as g:
                cf_exact_step(g, row_end, src, w, users, items, "cf %d users rank %d/%d" % (users, rank, world))
                x = O.cf_init(len(row_end))
                g.set_values(x)
                g.iterate(3)
                close(g.values().reshape(-1), O.colfilter(row_end, src, w, 3).reshape(-1), "cf 3 iterations rank %d" % rank, 2e-6)

    run_ranks(world, body)


def _bc_cases(world, weighted, big):
    mod = BW if weighted else B
    cases = []
    for fname, make in (("small_forest", mod.small_forest), ("forest", mod.forest))[:2 if big else 1]:
        f = make()
        cases.append((fname, f["row_end"], f["src"], f.get("weight"), f["roots"], f["scores"]))
    re14, src14 = graph("rmat14")
    w14 = W.rmat_weights(27, re14, src14) if weighted else None
    cases.append(("rmat14", re14, src14, w14, np.random.default_rng(14).choice(1 << 14, 6, replace=False).astype(np.uint32), None))
    re_t, src_t = edge_free_case(world)
    w_t = np.random.default_rng(5).integers(1, 256, len(src_t)).astype(np.int32) if weighted else None
    cases.append(("edge_free_last_rank", re_t, src_t, w_t, np.array([0, 3, 17, 499, len(re_t) - 1], np.uint32), None))
    return cases


def case_bc(world, weighted, big=False):
    cases = _bc_cases(world, weighted, big)
    refs = [(BW.run(r, s, w, src_) if weighted else B.run(r, s, src_)) for _, r, s, w, src_, _ in cases]

    def body(rank, uid):
        for i, ((name, row_end, src, w, sources, scores), ref) in enumerate(zip(cases, refs)):
            what = "%sbc %s rank %d/%d" % ("weighted " if weighted else "", name, rank, world)
            with opened(uid, i, world, rank, row_end, src, w, app=L.APP_BC_WEIGHTED if weighted else L.APP_BC) as g:
                b = g.bounds()
                if name == "edge_free_last_rank":
                    assert int(b["col_left"][-1]) == len(src) and int(b["row_right"][-1]) >= int(b["row_left"][-1]), what
                g.bc_run(sources)
                bc = g.values()
                lev, sigma, delta = g.bc_source_state()
            first_diff(lev, ref["dist"] if weighted else ref["lev"], what + " lev")
            first_diff(sigma, ref["sigma"], what + " sigma")
            if scores is not None:
                first_diff(delta, ref["delta"], what + " delta")
                first_diff(bc, scores, what + " scores")
            else:
                close(delta, ref["delta"], what + " delta", 1e-10)
                close(bc, ref["scores"], what + " scores", 1e-10)

    run_ranks(world, body)


def case_tc(world):
    cases = [("rmat14_device", None, None, False), ("rmat16 balanced", *graph("rmat16"), True),
             ("k300_both", *T.variant(*T.complete(300)[:2], "both"), False),
             ("edge_free_last_rank", *edge_free_case(world), False)]
    with L.LuxGraph.from_rmat(14, 1 << 14, 16 << 14, 5) as h:
        cases[0] = ("rmat14_device", *h.local_csc(), False)
    refs = [T.run(r, s) for _, r, s, _ in cases]

    def body(rank, uid):
        for i, ((name, row_end, src, balanced), ref) in enumerate(zip(cases, refs)):
            what = "tc %s rank %d/%d" % (name, rank, world)
            if name == "rmat14_device":
                g = L.LuxGraph.from_rmat(14, 1 << 14, 16 << 14, 5, app=L.APP_TC, rank=rank, nranks=world, device=0)
                g.comm_init(uid(i))
                g.init()
            else:
                g = opened(uid, i, world, rank, row_end, src, app=L.APP_TC, balanced=balanced)
            with g:
                b = g.bounds()
                if name == "edge_free_last_rank":
                    assert int(b["col_left"][-1]) == len(src) and int(b["row_right"][-1]) >= int(b["row_left"][-1]), what
                if balanced:  # the cost-balanced cuts are for the pull apps: TC keeps the reference's split
                    assert not g.work_bounds()["balanced"], what
                total = g.tc_run()
                t = g.values()
                lo, n = g.local_range()
                local = g.local_values()
            assert total == ref["total"], "%s: T = %d, want %d" % (what, total, ref["total"])
            first_diff(t, ref["t"], what + " t")
            first_diff(local, ref["t"][lo:lo + n], what + " local_values")

    run_ranks(world, body)


def case_uncut(world, names):
    """Graphs the reference partitioner cannot cut into `world` parts: every app runs on the partitions the library
    keeps (some without edges, some without vertices where nv < world), and each result equals the one-rank oracle."""
    plans = []
    for name in names:
        row_end, src = edge_free_case(world) if name == "edge_free_last_rank" else graph(name)
        if name != "edge_free_last_rank":
            assert parts(row_end, src, world) < world, "%s partitions into %d" % (name, world)
        nv = len(row_end)
        w = np.random.default_rng(3).integers(1, 256, len(src)).astype(np.int32)
        sources = np.unique(np.array([0, nv // 2, nv - 1], np.uint32))
        labels = [(app, start, reference(app, row_end, src, w, start)) for app, start in ((CC, 0), (SSSP, 0), (SSSP, nv - 1), (WSSSP, 0))]
        plans.append(dict(name=name, row_end=row_end, src=src, w=w, sources=sources, labels=labels,
                          cf=O.colfilter(row_end, src, w, 2), bc=B.run(row_end, src, sources), bcw=BW.run(row_end, src, w, sources),
                          tc=T.run(row_end, src)))

    def body(rank, uid):
        ids = iter(range(1 << 20))
        sizes = []
        for p in plans:
            row_end, src, w, sources = p["row_end"], p["src"], p["w"], p["sources"]
            nv = len(row_end)
            what = "%s rank %d/%d" % (p["name"], rank, world)
            with opened(uid, next(ids), world, rank, row_end, src) as g:
                sizes.append(g.local_range()[1])
                exact_steps(g, row_end, src, what + " pagerank")
            for app, start, ref in p["labels"]:
                with opened(uid, next(ids), world, rank, row_end, src, w if app == WSSSP else None, app=LAPP[app], start=start) as g:
                    assert g.run_to_convergence() == ref.iters, what
                    first_diff(g.values(), ref.labels[-1], "%s %s labels" % (what, app))
                    first_diff(g.trace()[0], ref.active, "%s %s active" % (what, app))
            with opened(uid, next(ids), world, rank, row_end, src, w, app=L.APP_COLFILTER) as g:
                g.set_values(O.cf_init(nv))
                g.iterate(2)
                close(g.values().reshape(-1), p["cf"].reshape(-1), what + " cf", 2e-6)
            with opened(uid, next(ids), world, rank, row_end, src, app=L.APP_BC) as g:
                g.bc_run(sources)
                close(g.values(), p["bc"]["scores"], what + " bc", 1e-10)
                first_diff(g.bc_source_state()[1], p["bc"]["sigma"], what + " bc sigma")
            with opened(uid, next(ids), world, rank, row_end, src, w, app=L.APP_BC_WEIGHTED) as g:
                g.bc_run(sources)
                close(g.values(), p["bcw"]["scores"], what + " weighted bc", 1e-10)
                lev, sigma, _ = g.bc_source_state()
                first_diff(lev, p["bcw"]["dist"], what + " weighted bc dist")
                first_diff(sigma, p["bcw"]["sigma"], what + " weighted bc sigma")
            with opened(uid, next(ids), world, rank, row_end, src, app=L.APP_TC) as g:
                assert g.tc_run() == p["tc"]["total"], what
                first_diff(g.values(), p["tc"]["t"], what + " tc")
        return sizes

    out = run_ranks(world, body)
    for i, p in enumerate(plans):
        if len(p["row_end"]) < world:  # the case the name promises: some ranks hold no vertex at all
            assert any(out[r][i] == 0 for r in range(world)), "%s: no rank without vertices" % p["name"]


def case_p2p_without_import(world):
    """exchange=P2P on handles that never import peer mappings: p2p_ready stays off and every exchange takes the NCCL
    path, with EXCHANGE_NCCL's results."""
    row_end, src = graph("rmat16")
    ref = O.label_run(O.APP_SSSP, row_end, src, P=world, start=0)

    def body(rank, uid):
        with opened(uid, 0, world, rank, row_end, src, exchange=L.EXCHANGE_P2P) as g:
            exact_steps(g, row_end, src, "pagerank p2p without import rank %d" % rank)
        with opened(uid, 1, world, rank, row_end, src, app=L.APP_SSSP, exchange=L.EXCHANGE_P2P) as g:
            assert g.run_to_convergence() == ref["iters"]
            first_diff(g.values(), ref["labels"], "sssp p2p without import rank %d" % rank)
            first_diff(g.trace()[0], ref["active"], "sssp p2p without import trace rank %d" % rank)

    run_ranks(world, body)


# ---- tests: each runs its case at every world in one subprocess -------------------------------------------------------
def run_case(case, worlds=WORLDS, env=None, **kw):
    rc, out = emulate("test_gpu_emulated_ranks", case, env=env, worlds=list(worlds), **kw)
    assert rc == 0, out[-6000:]


def test_partitions():
    run_case("case_partitions")


PR_GRAPHS = ["rmat16"] + sorted(ALL_SMALL)
PR_PATHS = {"seg": (dict(LUXB_SB=0), {}), "panel": (PANEL, dict(sweep="panel")),
            "merge": (dict(PANEL, LUXB_SWEEP="merge"), dict(sweep="merge")),
            "zero_copy": (PANEL, dict(zero_copy=True, sweep="merge")), "balanced": ({}, dict(balanced=True, sweep=None))}


@pytest.mark.parametrize("path", sorted(PR_PATHS))
def test_pagerank_exact_steps(path):
    env, kw = PR_PATHS[path]
    run_case("case_pagerank", env=env, names=PR_GRAPHS, **kw)


@pytest.mark.parametrize("group", ["cases", "fixtures", "bitmap"])
def test_labels_every_iteration_every_rank(group):
    run_case("case_labels", group=group, restart=group != "cases")


def test_labels_through_the_panel_split():
    run_case("case_labels", env=PANEL, group="bitmap")


def test_colfilter_exact_step():
    run_case("case_colfilter")


@pytest.mark.parametrize("weighted", [False, True])
def test_bc(weighted):
    run_case("case_bc", weighted=weighted)


@heavy
@pytest.mark.parametrize("weighted", [False, True])
def test_bc_large_forest(weighted):
    run_case("case_bc", [4], weighted=weighted, big=True)


def test_tc():
    run_case("case_tc", WORLDS + [8])


def test_partitions_the_reference_cannot_cut():
    run_case("case_uncut", names=["edge_free_last_rank", "hand5", "no_edges"])


def test_64_ranks():
    """LUXB_MAX_PARTS ranks on small graphs the reference cuts into fewer parts (every app), one with fewer vertices
    than ranks."""
    run_case("case_uncut", [64], names=["rmat12_ragged_nv", "star", "hand5"])


def test_p2p_exchange_without_import_takes_nccl():
    run_case("case_p2p_without_import", [2, 4])
