"""GPU: the CC / SSSP / weighted SSSP frontier engine (push.cuh, label_iteration and reset_label_state in api.cu)
pinned iteration by iteration.  After EVERY iterate(1) the label vector equals label_pull^k of the start labels, and
the active count, the frontier representation (stats()["last_frontier_type"]) and the newest trace entry equal the
oracle's.  The designed cases of tests/test_frontier_cases_model.py put a push or queue boundary in one iteration each
(big-source degrees around the inline / segment split, new frontiers around the queue capacity, the push / pull
threshold, demotion at capacity, exactly-once enqueue under contention, ragged and tiny nv); restarts through
set_values, resumed runs and iterations after convergence follow the same sequence."""
import numpy as np
import pytest

import lux_b200 as L
import weighted_oracle as W
from test_frontier_cases_model import (CASE_RUNS, CC, FIXTURE_RUNS, NV, SSSP, WSSSP, assert_jacobi_is_the_oracle, build_run,
                                       case_run_id, jacobi, reference)

pytestmark = pytest.mark.gpu
LAPP = {CC: L.APP_CC, SSSP: L.APP_SSSP, WSSSP: L.APP_SSSP_WEIGHTED}


def open_graph(app, row_end, src, w, start):
    return L.LuxGraph.from_csc(row_end, src, w if app == WSSSP else None, app=LAPP[app], start=start)


def step(g, ref, n=None, what=""):
    """iterate(1) n times (default: through the iteration that reports 0 active), checking after each one the labels
    against ref.labels[k + 1], the returned active count, stats() and the newest trace entry."""
    n = ref.iters if n is None else n
    base = len(g.trace()[0])
    for k in range(n):
        act = g.iterate(1)
        lab = g.values()
        bad = np.nonzero(lab != ref.labels[k + 1])[0]
        assert len(bad) == 0, "%s iteration %d: %d labels differ, first at %s" % (what, k, len(bad), bad[:8])
        assert act == ref.active[k], "%s iteration %d: active %d, want %d" % (what, k, act, ref.active[k])
        st = g.stats()
        assert st["last_active"] == ref.active[k]
        assert st["last_frontier_type"] == ref.ftype[k], "%s iteration %d (active %d): frontier type %#x, want %#x" % (
            what, k, act, st["last_frontier_type"], ref.ftype[k])
        a, p = g.trace()
        assert len(a) == base + k + 1
        assert (a[-1], p[-1]) == (ref.active[k], ref.pull[k]), "%s iteration %d: trace entry" % (what, k)


@pytest.mark.parametrize("run", CASE_RUNS + FIXTURE_RUNS, ids=case_run_id)
def test_every_iteration_matches_the_oracle(run):
    name, app, start = run
    row_end, src, w, _ = build_run(name)
    ref = assert_jacobi_is_the_oracle(app, row_end, src, w, start)
    with open_graph(app, row_end, src, w, start) as g:
        g.init()
        step(g, ref, what=case_run_id(run))
        assert g.stats()["iterations"] == ref.iters
        assert g.check() == 0
    with open_graph(app, row_end, src, w, start) as g:
        g.init()
        assert g.run_to_convergence() == ref.iters
        assert np.array_equal(g.values(), ref.labels[-1])
        active, pull = g.trace()
        assert np.array_equal(active, ref.active) and np.array_equal(pull, ref.pull)
        assert g.stats()["last_frontier_type"] == ref.ftype[-1]


RESTART_RUNS = [("rmat14_sym", CC, 0), ("rmat14", SSSP, 0), ("rmat14", WSSSP, 0),
                ("queue_at_capacity_many_+0", CC, 0), ("queue_at_capacity_many_+0", SSSP, NV - 1),
                ("queue_at_capacity_many_+0", WSSSP, NV - 1)]


@pytest.mark.parametrize("run", RESTART_RUNS, ids=case_run_id)
def test_checkpoint_restart_continues_the_run(run):
    """set_values(L_k) after k iterations makes every vertex active (a dense frontier of nv), and the run goes on as
    label_pull^j(L_k) to the uninterrupted fixpoint; the trace keeps appending."""
    name, app, start = run
    row_end, src, w, _ = build_run(name)
    nv = len(row_end)
    ref = reference(app, row_end, src, w, start)
    assert ref.iters >= 3
    for k in sorted({1, ref.iters // 2, ref.iters - 1}):
        with open_graph(app, row_end, src, w, start) as g:
            g.init()
            step(g, ref, n=k, what="before restart")
            g.set_values(ref.labels[k])
            st = g.stats()
            assert st["last_active"] == nv and st["last_frontier_type"] == L.DENSE_BITMAP
            again = jacobi(app, row_end, src, w, ref.labels[k], nv)
            assert again.pull[0] == 1
            step(g, again, what="restart at %d" % k)
            assert np.array_equal(g.values(), ref.labels[-1])
            assert len(g.trace()[0]) == k + again.iters
            assert g.check() == 0


@pytest.mark.parametrize("run", RESTART_RUNS, ids=case_run_id)
def test_restart_from_arbitrary_labels(run):
    """set_values of labels that are not a checkpoint (SSSP: the fixpoint plus random increments, clipped to INF; CC:
    random labels): the run is label_pull iterated from them, iteration by iteration, to a state check() accepts."""
    name, app, start = run
    row_end, src, w, _ = build_run(name)
    nv = len(row_end)
    rng = np.random.default_rng(17)
    if app == CC:
        lab0 = rng.integers(0, nv, nv).astype(np.uint32)
    else:
        inf = nv if app == SSSP else W.INF
        fix = reference(app, row_end, src, w, start).labels[-1].astype(np.int64)
        lab0 = np.minimum(fix + rng.integers(0, 4 if app == SSSP else 40, nv), inf).astype(np.uint32)
    ref = jacobi(app, row_end, src, w, lab0, nv)
    assert ref.iters >= 2
    with open_graph(app, row_end, src, w, start) as g:
        g.init()
        g.set_values(lab0)
        st = g.stats()
        assert st["last_active"] == nv and st["last_frontier_type"] == L.DENSE_BITMAP
        step(g, ref, what="arbitrary restart")
        assert g.check() == 0


@pytest.mark.parametrize("run", RESTART_RUNS, ids=case_run_id)
def test_resume_and_iterate_after_convergence(run):
    """run_to_convergence(max_iters=k) then run_to_convergence() is the uninterrupted run (labels, concatenated
    trace); iterate(3) after convergence reports 0 active and changes no label."""
    name, app, start = run
    row_end, src, w, _ = build_run(name)
    ref = reference(app, row_end, src, w, start)
    k = max(1, ref.iters // 2)
    with open_graph(app, row_end, src, w, start) as g:
        g.init()
        assert g.run_to_convergence(max_iters=k) == k
        assert np.array_equal(g.values(), ref.labels[k])
        assert g.run_to_convergence() == ref.iters - k
        lab = g.values()
        assert np.array_equal(lab, ref.labels[-1])
        active, pull = g.trace()
        assert np.array_equal(active, ref.active) and np.array_equal(pull, ref.pull)
        assert g.iterate(3) == 0
        assert np.array_equal(g.values(), lab)
        assert g.stats()["last_active"] == 0 and g.check() == 0
