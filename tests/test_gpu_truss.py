"""GPU parity of the k-truss decomposition (LUXB_TRUSS) against the CPU oracle tests/truss_oracle.c, which
tests/test_truss_oracle.py pins to networkx, scipy, its own two peels and closed forms.  Integers only and a
deterministic round structure, so everything is bit for bit: the edges, support and τ (truss_edges()), the vertex truss
(values()), kmax, stats.iterations == rounds, the round trace (|F|, k), stats.edges_processed == m per run and
check() == 0.  Exact families: K_2048 under storage noise, disjoint cliques K_3 .. K_30, a book of 2^17 pages (the spine
takes 2^17 decrements in one round), a wheel, K_{p,q}, a cycle, a grid, a triangulated tube of 3000 rounds, a graph
without edges and triangle counting's over-budget graph (out-lists longer than kTcSharedList: the big kernel counts the
support).  Also the configurations, repeat runs, check() on planted corruptions, error codes, the public surfaces and
several ranks on one device through the in-process NCCL stand-in (tests/emu_ranks.py) and several GPUs.
LUXB_SKIP_HEAVY=1 skips RMAT-18 (the oracle's sequential peels take minutes there)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import lux_b200 as L
import tc_oracle as T
import truss_oracle as R
from emu_ranks import emulate, run_ranks
from graphs import ALL_SMALL, rmat
from mgpu_bc_worker import edge_free_case
from test_gpu_emulated_ranks import first_diff, opened

pytestmark = pytest.mark.gpu
heavy = pytest.mark.skipif(os.environ.get("LUXB_SKIP_HEAVY") == "1", reason="LUXB_SKIP_HEAVY=1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUDGET = 1024  # kTcSharedList (tc.cuh)


def assert_matches(g, ref, what, runs=1):
    """A handle after `runs` runs: edges, support, τ, vertex truss, trace, stats and check() against the oracle."""
    lo, hi, sup, tau = g.truss_edges()
    first_diff(lo, ref["lo"], what + " lo")
    first_diff(hi, ref["hi"], what + " hi")
    first_diff(sup, ref["support"], what + " support")
    first_diff(tau, ref["truss"], what + " truss")
    tv = g.values()
    assert tv.dtype == np.uint32
    first_diff(tv, ref["vertex"], what + " vertex truss")
    active, pull = g.trace()
    first_diff(active, ref["trace_active"], what + " trace |F|")
    first_diff(pull, ref["trace_k"], what + " trace k")
    st = g.stats()
    assert st["iterations"] == runs * ref["rounds"], what
    assert st["edges_processed"] == runs * ref["m"], what
    assert g.check() == 0, what


def check(row_end, src, want=None, ref=None, **kw):
    ref = R.run(row_end, src) if ref is None else ref
    if want is not None:
        assert np.array_equal(ref["truss"], want)
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_TRUSS, **kw) as g:
        g.init()
        assert g.truss_num_edges() == ref["m"]
        assert g.truss_run() == ref["kmax"]
        assert_matches(g, ref, "truss")
    return ref


@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_small_fixtures(name):
    check(*ALL_SMALL[name]())


@pytest.mark.parametrize("scale", [10, 12, 14, 16, pytest.param(18, marks=heavy)])
def test_rmat(scale):
    ref = check(*rmat(scale))
    assert ref["kmax"] > 2 and ref["rounds"] > ref["levels"]


@pytest.mark.parametrize("kind", T.VARIANTS)
def test_k2048_noise(kind):
    row_end, src, tau = R.complete(2048)
    check(*T.variant(row_end, src, kind, seed=3), want=tau, ref=R.clique_result(2048))


@pytest.mark.parametrize("name", sorted(R.CLOSED_FORMS))
def test_closed_forms(name):
    row_end, src, tau = R.CLOSED_FORMS[name]()
    check(row_end, src, want=tau)


def test_support_over_budget():
    row_end, src, _ = T.over_budget(BUDGET, 3)
    ref = check(row_end, src)
    assert ref["kmax"] >= 3


def test_zero_copy_edges():
    check(*rmat(14), zero_copy=True)


def test_weighted_csc_accepted():
    row_end, src = rmat(12)
    check(row_end, src, weight=np.arange(len(src), dtype=np.int32) % 7 - 3)


def test_rmat_generated_on_device():
    with L.LuxGraph.from_rmat(14, 1 << 14, 16 << 14, 11, app=L.APP_TRUSS) as g:
        row_end, src = g.local_csc()
        g.init()
        kmax = g.truss_run()
        ref = R.run(row_end, src)
        assert kmax == ref["kmax"]
        assert_matches(g, ref, "device rmat14")
        first_diff(g.local_values(), ref["vertex"], "device rmat14 local_values")


def test_two_runs_and_values():
    row_end, src = rmat(13)
    ref = R.run(row_end, src)
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_TRUSS) as g:
        g.init()
        assert not g.values().any()  # zeros before the first run
        lo, hi, sup, tau = g.truss_edges()
        assert not tau.any() and np.array_equal(sup, ref["support"])  # the support is there from luxb_init
        assert g.truss_run() == ref["kmax"]
        g.set_truss(np.zeros(ref["m"], np.uint32))  # the next run recomputes from scratch
        assert not g.values().any()
        assert g.truss_run() == ref["kmax"]
        assert_matches(g, ref, "second run", runs=2)
        assert g.stats()["loop_seconds"] > 0


def test_check_on_planted_corruptions():
    row_end, src = rmat(12)
    ref = R.run(row_end, src)
    good = ref["truss"]
    rng = np.random.default_rng(4)
    cases = []
    for e in rng.choice(len(good), 4, replace=False):
        for d in (1, -1):
            bad = good.copy()
            bad[e] = int(good[e]) + d
            cases.append(bad)
    cases += [rng.permutation(good), np.full_like(good, 0xFFFFFFFF)]
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_TRUSS) as g:
        g.init()
        g.truss_run()
        for tau in cases:
            g.set_truss(tau)
            assert g.check() == R.check(row_end, src, tau)[0]
            tv = np.zeros(len(row_end), np.uint32)
            np.maximum.at(tv, ref["lo"], tau)
            np.maximum.at(tv, ref["hi"], tau)
            first_diff(g.values(), tv, "vertex truss after set_truss")
        assert g.check() > 0
        g.set_truss(np.full_like(good, 2))
        assert g.check() == 0  # all 2s pass: the check is necessary, not sufficient
        g.truss_run()
        first_diff(g.truss_edges()[3], good, "run after set_truss")


def test_errors():
    row_end, src = rmat(10)
    nv = len(row_end)
    lib = L.load_library()
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_TRUSS) as g:
        with pytest.raises(L.LuxError, match=r"\(-5\)"):   # before luxb_init
            g.truss_run()
        g.init()
        g.truss_run()
        m = g.truss_num_edges()
        before = g.values()
        for call in (lambda: g.iterate(1), lambda: g.run_to_convergence(), lambda: g.set_values(np.zeros(nv, np.uint32)),
                     lambda: g.set_local_values(np.zeros(nv, np.uint32))):
            with pytest.raises(L.LuxError, match=r"\(-1\).*luxb_truss_run"):
                call()
        with pytest.raises(L.LuxError, match=r"\(-1\)"):
            g.kcore_run()
        with pytest.raises(L.LuxError, match=r"\(-1\)"):
            g.set_truss(np.zeros(m + 1, np.uint32))
        z = np.zeros(m - 1, np.uint32)
        assert lib.luxb_truss_edges(g._h, None, None, None, z.ctypes.data_as(L.binding.C.c_void_p), L.binding.C.c_uint64(m - 1)) == -1
        assert lib.luxb_truss_edges(g._h, None, None, None, None, L.binding.C.c_uint64(m)) == 0  # NULL skips
        assert np.array_equal(g.values(), before)
        assert lib.luxb_truss_run(g._h, None) == 0  # kmax is optional
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_KCORE) as g:
        g.init()
        for call in (g.truss_run, g.truss_num_edges, lambda: g.set_truss(np.zeros(1, np.uint32))):
            with pytest.raises(L.LuxError, match=r"\(-1\)"):
                call()


def test_apps_and_torch_op():
    import torch
    import lux_b200.torch_ops  # noqa: F401
    row_end, src = rmat(11)
    ref = R.run(row_end, src)
    out = L.truss(row_end, src)
    assert out["kmax"] == ref["kmax"] and out["rounds"] == ref["rounds"]
    for key in ("lo", "hi", "support", "truss", "vertex"):
        first_diff(out[key], ref[key], "apps.truss " + key)
    edges, tau = torch.ops.luxb.k_truss(torch.from_numpy(row_end.astype(np.int64)).cuda(), torch.from_numpy(src.astype(np.int64)).cuda())
    assert edges.dtype == torch.int64 and tau.dtype == torch.int64 and edges.is_cuda and edges.shape == (ref["m"], 2)
    assert np.array_equal(edges.cpu().numpy(), np.stack([ref["lo"], ref["hi"]], 1).astype(np.int64))
    assert np.array_equal(tau.cpu().numpy(), ref["truss"].astype(np.int64))


def test_cli(tmp_path):
    row_end, src = rmat(11)
    path = str(tmp_path / "g.lux")
    L.write_lux(path, row_end, src)
    out = str(tmp_path / "truss.npz")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "apps", "lux_cli.py"), "truss", "-file", path, "-check", "-out", out],
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    ref = R.run(row_end, src)
    assert re.search(r"ELAPSED TIME = \d", p.stdout) and "[Memory Setting]" not in p.stdout
    assert re.search(r"^KMAX = %d$" % ref["kmax"], p.stdout, re.M)
    assert re.search(r"^\[PASS\] Check task: rowLeft\(0\) numMistakes\(0\)$", p.stdout, re.M)
    z = np.load(out)
    for key in ("lo", "hi", "support", "truss", "vertex"):
        assert z[key].dtype == np.uint32 and np.array_equal(z[key], ref[key]), key


# ---- several ranks on one device (in-process NCCL stand-in) -----------------------------------------------------------
EMU_CLOSED = {"k48": lambda: R.complete(48), "cliques": lambda: R.cliques(20), "book": lambda: R.book(1 << 12),
              "wheel": lambda: R.wheel(300), "grid": lambda: R.grid(20, 30), "tube": lambda: R.tube(200),
              "no_edges": lambda: R.no_edges()}


def _graph(name, world):
    if name == "edge_free_last_rank":
        return edge_free_case(world)
    if name in EMU_CLOSED:
        return EMU_CLOSED[name]()[:2]
    if name in ALL_SMALL:
        return ALL_SMALL[name]()
    return rmat(int(name[4:]))


def case_truss(world, names):
    """Every rank's edges, support, τ, vertex truss, local_values(), kmax, stats and trace against the one-rank oracle;
    check() summed over the ranks is 0 on the result and equals the oracle's count on a corrupted assignment."""
    plans = []
    for name in names:
        row_end, src = _graph(name, world)
        ref = R.run(row_end, src)
        bad = ref["truss"].copy()
        if len(bad):
            bad[np.argmax(bad)] += 1
        plans.append((name, row_end, src, ref, bad, R.check(row_end, src, bad)[0]))

    def body(rank, uid):
        checks = []
        for i, (name, row_end, src, ref, bad, _) in enumerate(plans):
            what = "truss %s rank %d/%d" % (name, rank, world)
            with opened(uid, i, world, rank, row_end, src, app=L.APP_TRUSS) as g:
                if name == "edge_free_last_rank":
                    b = g.bounds()
                    assert int(b["col_left"][-1]) == len(src) and int(b["row_right"][-1]) >= int(b["row_left"][-1]), what
                assert g.truss_run() == ref["kmax"], what
                assert_matches(g, ref, what)
                lo, n = g.local_range()
                first_diff(g.local_values(), ref["vertex"][lo:lo + n], what + " local_values")
                good = g.check()
                g.set_truss(bad)
                checks.append((good, g.check()))
        return checks

    out = run_ranks(world, body)
    for i, (name, _, _, _, _, want_bad) in enumerate(plans):
        assert sum(out[r][i][0] for r in range(world)) == 0, name
        assert sum(out[r][i][1] for r in range(world)) == want_bad, "%s: check over the ranks" % name


def run_case(worlds, names):
    rc, out = emulate("test_gpu_truss", "case_truss", worlds=list(worlds), names=list(names))
    assert rc == 0, out[-6000:]


@pytest.mark.parametrize("names", [["rmat12", "rmat14"], sorted(EMU_CLOSED) + ["edge_free_last_rank"]], ids=["rmat", "closed"])
def test_emulated_ranks(names):
    run_case([2, 3, 4, 8], names)


def test_emulated_64_ranks():
    """64 ranks on small graphs, one with fewer vertices than ranks (ranks without vertices)."""
    assert len(ALL_SMALL["hand5"]()[0]) < 64
    run_case([64], ["hand5", "book", "rmat12_ragged_nv", "no_edges"])


# ---- several GPUs (real NCCL) -------------------------------------------------------------------------------------------
def _run_worker(world, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mgpu_truss_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    return p.returncode, p.stdout + p.stderr


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_truss(world, gpu_count):
    if gpu_count < world:
        pytest.skip("needs %d GPUs, have %d" % (world, gpu_count))
    rc, out = _run_worker(world, 29640 + world)
    assert rc == 0 and "MGPU_TRUSS PASS" in out, out[-4000:]
