"""GPU parity of the k-core decomposition (LUXB_KCORE) against the CPU oracle tests/kcore_oracle.c, which
tests/test_kcore_oracle.py pins to networkx, a numpy restatement of the schedule and closed forms.  Integers only and a
deterministic round structure, so everything is bit for bit: core, the degeneracy, stats.iterations == rounds, the round
trace (|F|, k), stats.edges_processed == 2m per run, and check() == 0.  Exact families need no oracle: K_2048 under
storage noise, K_{p,q}, a cycle and a grid, a star whose hub takes 2^17 concurrent decrements, a 3001-vertex path (1501
rounds at one level), a chain of cliques K_2 .. K_200 (199 levels) and a clique with a hub of 2^17 leaves.  Also the
configurations, repeat runs, check() on planted corruptions, error codes, the public surfaces, C4 at full size, several
ranks on one device through the in-process NCCL stand-in (tests/emu_ranks.py) and several GPUs.  LUXB_SKIP_HEAVY=1
skips C4."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import kcore_oracle as K
import lux_b200 as L
import tc_oracle as T
from emu_ranks import emulate, run_ranks
from graphs import ALL_SMALL, rmat
from mgpu_bc_worker import edge_free_case
from test_gpu_emulated_ranks import first_diff, opened

pytestmark = pytest.mark.gpu
heavy = pytest.mark.skipif(os.environ.get("LUXB_SKIP_HEAVY") == "1", reason="LUXB_SKIP_HEAVY=1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def assert_matches(g, ref, what, runs=1):
    """A handle after `runs` runs: core, trace, stats and check() against the oracle's result."""
    core = g.values()
    assert core.dtype == np.uint32
    first_diff(core, ref["core"], what + " core")
    active, pull = g.trace()
    first_diff(active, ref["trace_active"], what + " trace |F|")
    first_diff(pull, ref["trace_k"], what + " trace k")
    st = g.stats()
    assert st["iterations"] == runs * ref["rounds"], what
    assert st["edges_processed"] == runs * 2 * ref["m"], what
    assert g.check() == 0, what


def check(row_end, src, want=None, **kw):
    ref = K.run(row_end, src)
    if want is not None:
        assert np.array_equal(ref["core"], want)
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_KCORE, **kw) as g:
        g.init()
        assert g.kcore_run() == ref["degeneracy"]
        assert_matches(g, ref, "kcore")
    return ref


@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_small_fixtures(name):
    check(*ALL_SMALL[name]())


@pytest.mark.parametrize("scale", [10, 12, 14, 16, 18])
def test_rmat(scale):
    ref = check(*rmat(scale))
    assert ref["degeneracy"] > 0 and ref["rounds"] > ref["levels"]


@pytest.mark.parametrize("kind", T.VARIANTS)
def test_k2048_noise(kind):
    row_end, src, core = K.complete(2048)
    check(*T.variant(row_end, src, kind, seed=3), want=core)


@pytest.mark.parametrize("name", sorted(K.CLOSED_FORMS))
def test_closed_forms(name):
    row_end, src, core = K.CLOSED_FORMS[name]()
    check(row_end, src, want=core)


def test_zero_copy_edges():
    check(*rmat(15), zero_copy=True)


def test_weighted_csc_accepted():
    row_end, src = rmat(12)
    check(row_end, src, weight=np.arange(len(src), dtype=np.int32) % 7 - 3)


def test_rmat_generated_on_device():
    with L.LuxGraph.from_rmat(15, 1 << 15, 16 << 15, 11, app=L.APP_KCORE) as g:
        row_end, src = g.local_csc()
        g.init()
        degeneracy = g.kcore_run()
        ref = K.run(row_end, src)
        assert degeneracy == ref["degeneracy"]
        assert_matches(g, ref, "device rmat15")
        first_diff(g.local_values(), ref["core"], "device rmat15 local_values")


def test_two_runs_and_values():
    row_end, src = rmat(14)
    ref = K.run(row_end, src)
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_KCORE) as g:
        g.init()
        assert not g.values().any()  # zeros before the first run
        assert g.kcore_run() == ref["degeneracy"]
        first = g.values()
        g.set_values(np.zeros(len(row_end), np.uint32))  # the next run recomputes from scratch
        assert g.kcore_run() == ref["degeneracy"]
        assert np.array_equal(first, g.values())
        assert_matches(g, ref, "second run", runs=2)
        assert g.stats()["loop_seconds"] > 0


def test_check_on_planted_corruptions():
    row_end, src = rmat(13)
    ref = K.run(row_end, src)
    good = ref["core"]
    rng = np.random.default_rng(4)
    cases = []
    for v in rng.choice(np.nonzero(good > 0)[0], 4, replace=False):
        for d in (1, -1):
            bad = good.copy()
            bad[v] = int(good[v]) + d
            cases.append(bad)
    cases += [rng.permutation(good), np.zeros_like(good), np.full_like(good, 0xFFFFFFFF)]
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_KCORE) as g:
        g.init()
        g.kcore_run()
        for core in cases:
            g.set_values(core)
            assert g.check() == K.check(row_end, src, core)[0]
        assert g.check() > 0
        g.set_values(np.zeros_like(good))
        assert g.check() == 0  # all zeros pass: the check is necessary, not sufficient
        g.kcore_run()
        first_diff(g.values(), good, "run after set_values")


def test_errors():
    row_end, src = rmat(10)
    nv = len(row_end)
    lib = L.load_library()
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_KCORE) as g:
        with pytest.raises(L.LuxError, match=r"\(-5\)"):   # before luxb_init
            g.kcore_run()
        g.init()
        g.kcore_run()
        before = g.values()
        for call in (lambda: g.iterate(1), lambda: g.run_to_convergence()):
            with pytest.raises(L.LuxError, match=r"\(-1\).*luxb_kcore_run"):
                call()
        with pytest.raises(L.LuxError, match=r"\(-1\)"):
            g.tc_run()
        with pytest.raises(L.LuxError, match=r"\(-1\)"):
            g.set_values(np.zeros(nv + 1, np.uint32))
        assert np.array_equal(g.values(), before)
        assert lib.luxb_kcore_run(g._h, None) == 0  # the degeneracy is optional
        assert not g.work_bounds()["balanced"]
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_TC) as g:
        g.init()
        with pytest.raises(L.LuxError, match=r"\(-1\)"):
            g.kcore_run()


def test_apps_and_torch_op():
    import torch
    import lux_b200.torch_ops  # noqa: F401
    row_end, src = rmat(11)
    ref = K.run(row_end, src)
    out = L.core_number(row_end, src)
    assert out["degeneracy"] == ref["degeneracy"] and out["rounds"] == ref["rounds"]
    first_diff(out["core"], ref["core"], "apps.core_number")
    c = torch.ops.luxb.core_number(torch.from_numpy(row_end.astype(np.int64)).cuda(), torch.from_numpy(src.astype(np.int64)).cuda())
    assert c.dtype == torch.int64 and c.is_cuda and c.shape == (len(row_end),)
    assert np.array_equal(c.cpu().numpy(), ref["core"].astype(np.int64))


def test_cli(tmp_path):
    row_end, src = rmat(11)
    path = str(tmp_path / "g.lux")
    L.write_lux(path, row_end, src)
    out = str(tmp_path / "core.npy")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "apps", "lux_cli.py"), "kcore", "-file", path, "-check", "-out", out],
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    ref = K.run(row_end, src)
    assert re.search(r"ELAPSED TIME = \d", p.stdout) and "[Memory Setting]" not in p.stdout
    assert re.search(r"^DEGENERACY = %d$" % ref["degeneracy"], p.stdout, re.M)
    assert re.search(r"^\[PASS\] Check task: rowLeft\(0\) numMistakes\(0\)$", p.stdout, re.M)
    core = np.load(out)
    assert core.dtype == np.uint32 and np.array_equal(core, ref["core"])


@heavy
def test_c4_rmat24():
    from test_gpu_configs import check_blocks_against_oracle_generator, scale_of
    nv, ne, seed = 1 << 24, 16 << 24, 24
    with L.LuxGraph.from_rmat(scale_of(nv), nv, ne, seed, app=L.APP_KCORE) as g:
        row_end, src = g.local_csc()
        g.init()
        degeneracy = g.kcore_run()
        check_blocks_against_oracle_generator(scale_of(nv), nv, ne, seed, row_end, src)
        ref = K.run(row_end, src)
        assert degeneracy == ref["degeneracy"]
        assert_matches(g, ref, "C4")
    print("C4 k-core: degeneracy %d, %d levels, %d rounds, widest round %d, m = %d" % (
        ref["degeneracy"], ref["levels"], ref["rounds"], ref["max_frontier"], ref["m"]))


# ---- several ranks on one device (in-process NCCL stand-in) -----------------------------------------------------------
EMU_CLOSED = {"k64": lambda: K.complete(64), "k_30_45": lambda: K.complete_bipartite(30, 45), "grid": lambda: K.grid(40, 60),
              "star": lambda: K.star(1 << 14), "path": lambda: K.path(301), "clique_chain": lambda: K.clique_chain(2, 60),
              "hub_clique": lambda: K.hub_clique(101, 1 << 12)}


def _graph(name, world):
    if name == "edge_free_last_rank":
        return edge_free_case(world)
    if name in EMU_CLOSED:
        return EMU_CLOSED[name]()[:2]
    if name in ALL_SMALL:
        return ALL_SMALL[name]()
    return rmat(int(name[4:]))


def case_kcore(world, names):
    """Every rank's core numbers, local_values(), degeneracy, stats and trace against the one-rank oracle; check()
    summed over the ranks is 0 on the result and equals the oracle's count on a corrupted assignment."""
    plans = []
    for name in names:
        row_end, src = _graph(name, world)
        ref = K.run(row_end, src)
        bad = ref["core"].copy()
        bad[np.argmax(ref["core"])] += 1
        plans.append((name, row_end, src, ref, bad, K.check(row_end, src, bad)[0]))

    def body(rank, uid):
        checks = []
        for i, (name, row_end, src, ref, bad, _) in enumerate(plans):
            what = "kcore %s rank %d/%d" % (name, rank, world)
            with opened(uid, i, world, rank, row_end, src, app=L.APP_KCORE) as g:
                if name == "edge_free_last_rank":
                    b = g.bounds()
                    assert int(b["col_left"][-1]) == len(src) and int(b["row_right"][-1]) >= int(b["row_left"][-1]), what
                assert g.kcore_run() == ref["degeneracy"], what
                assert_matches(g, ref, what)
                lo, n = g.local_range()
                first_diff(g.local_values(), ref["core"][lo:lo + n], what + " local_values")
                good = g.check()
                g.set_values(bad)
                checks.append((good, g.check()))
        return checks

    out = run_ranks(world, body)
    for i, (name, _, _, _, _, want_bad) in enumerate(plans):
        assert sum(out[r][i][0] for r in range(world)) == 0, name
        assert sum(out[r][i][1] for r in range(world)) == want_bad, "%s: check over the ranks" % name


def run_case(worlds, names):
    rc, out = emulate("test_gpu_kcore", "case_kcore", worlds=list(worlds), names=list(names))
    assert rc == 0, out[-6000:]


@pytest.mark.parametrize("names", [["rmat14", "rmat16"], sorted(EMU_CLOSED) + ["edge_free_last_rank"]], ids=["rmat", "closed"])
def test_emulated_ranks(names):
    run_case([2, 3, 4, 8], names)


def test_emulated_64_ranks():
    """64 ranks on small graphs, one with fewer vertices than ranks (ranks without vertices)."""
    assert len(ALL_SMALL["hand5"]()[0]) < 64
    run_case([64], ["hand5", "star", "rmat12_ragged_nv", "no_edges"])


# ---- several GPUs (real NCCL) -------------------------------------------------------------------------------------------
def _run_worker(world, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mgpu_kcore_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    return p.returncode, p.stdout + p.stderr


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_kcore(world, gpu_count):
    if gpu_count < world:
        pytest.skip("needs %d GPUs, have %d" % (world, gpu_count))
    rc, out = _run_worker(world, 29630 + world)
    assert rc == 0 and "MGPU_KCORE PASS" in out, out[-4000:]
