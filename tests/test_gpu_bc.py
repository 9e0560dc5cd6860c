"""GPU parity of betweenness centrality (LUXB_BC) against the CPU oracle tests/bc_oracle.c, which tests/test_bc_oracle.py
pins to networkx and to hand-worked graphs.  Per source: the hop levels and the path counts sigma bit for bit (the
oracle's sigma < 2^53 is asserted, so both are exact integers), delta and the scores within rtol 1e-10 with exact
zeros.  On the forest inputs (bc_oracle.forest) every summation order is exact: delta and scores bit for bit, through
both split paths (a 2^17-child hub cuts the delta sum into segments, a vertex with 2^20 non-matching in-edges the sigma
sum).  Also: the BFS trace, one-rank reproducibility, the sweep configurations, C4 at full size, error codes, the public
surfaces and several GPUs.  LUXB_SKIP_HEAVY=1 skips C4."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
import lux_b200 as L
import bc_oracle as B
from graphs import ALL_SMALL, rmat

pytestmark = pytest.mark.gpu
heavy = pytest.mark.skipif(os.environ.get("LUXB_SKIP_HEAVY") == "1", reason="LUXB_SKIP_HEAVY=1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEEP = {"chain", "two_components"}  # up to 3000 levels per source: a level costs a few launches, so sources are sampled


def close(got, want, rtol=1e-10):
    assert np.array_equal(got == 0, want == 0), "zeros differ at %s" % np.nonzero((got == 0) != (want == 0))[0][:10]
    np.testing.assert_allclose(got, want, rtol=rtol, atol=0)


def check_state(g, ref_lev, ref_sigma, ref_delta):
    lev, sigma, delta = g.bc_source_state()
    assert ref_sigma.max() < 2.0 ** 53, "the oracle's sigma is no longer an exact integer"
    assert np.array_equal(lev, ref_lev), "levels differ at %s" % np.nonzero(lev != ref_lev)[0][:10]
    assert np.array_equal(sigma, ref_sigma), "sigma differs at %s" % np.nonzero(sigma != ref_sigma)[0][:10]
    close(delta, ref_delta)
    return lev, sigma, delta


def sources_for(name, nv):
    if nv <= 4096 and name not in DEEP:
        return np.arange(nv, dtype=np.uint32)
    return np.unique(np.concatenate([[0, nv - 1], np.random.default_rng(1).choice(nv, 24, replace=False)])).astype(np.uint32)


def per_source_parity(row_end, src, sources, **kw):
    """One handle, one bc_run per source: every source's state against the oracle, then the summed scores."""
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_BC, **kw) as g:
        g.init()
        for s in sources:
            g.bc_run([s])
            check_state(g, *B.source_state(row_end, src, s))
        bc = g.values()
        st = g.stats()
    close(bc, B.scores(row_end, src, sources))
    return st


@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_small_fixtures(name):
    row_end, src = ALL_SMALL[name]()
    per_source_parity(row_end, src, sources_for(name, len(row_end)))


@pytest.mark.parametrize("scale", [14, 16])
def test_rmat_sampled_sources(scale):
    row_end, src = rmat(scale)
    sources = np.random.default_rng(scale).choice(len(row_end), 8, replace=False).astype(np.uint32)
    st = per_source_parity(row_end, src, sources)
    assert st["iterations"] >= 8 and st["edges_processed"] > 0


def run_bc(row_end, src, sources, **kw):
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_BC, **kw) as g:
        g.init()
        g.bc_run(sources)
        return g.values(), g.bc_source_state(), g.trace(), g.stats()


@pytest.mark.parametrize("make", [B.small_forest, B.forest])
@pytest.mark.parametrize("config", ["default", "merge", "zero_copy"])
def test_exact_forest(make, config, monkeypatch):
    if config == "merge":
        monkeypatch.setenv("LUXB_SWEEP", "merge")
    f = make()
    ref = B.run(f["row_end"], f["src"], f["roots"])
    bc, (lev, sigma, delta), _, _ = run_bc(f["row_end"], f["src"], f["roots"], zero_copy=config == "zero_copy")
    assert np.array_equal(bc, f["scores"]) and np.array_equal(bc, ref["scores"])
    assert np.array_equal(lev, ref["lev"]) and np.array_equal(sigma, ref["sigma"]) and np.array_equal(delta, ref["delta"])


@pytest.mark.parametrize("config", ["merge", "zero_copy"])
def test_configurations_rmat(config, monkeypatch):
    if config == "merge":
        monkeypatch.setenv("LUXB_SWEEP", "merge")
    row_end, src = rmat(15)
    sources = np.random.default_rng(3).choice(len(row_end), 4, replace=False).astype(np.uint32)
    per_source_parity(row_end, src, sources, zero_copy=config == "zero_copy")


def test_bfs_trace_is_the_sssp_trace():
    row_end, src = rmat(16)
    for s in (0, 12345):
        _, (lev, _, _), (active, pull), _ = run_bc(row_end, src, [7, s])
        ref = O.label_run(O.APP_SSSP, row_end, src, start=s)
        assert np.array_equal(lev, ref["labels"])
        assert np.array_equal(active, ref["active"]) and np.array_equal(pull, ref["pull"])
        assert pull.sum() > 0  # the pull direction took part


def test_one_rank_is_bitwise_reproducible():
    row_end, src = rmat(15)
    a, b = 11, 2024
    bc1, _, _, _ = run_bc(row_end, src, [a, b])
    bc2, _, _, _ = run_bc(row_end, src, [a, b])
    assert np.array_equal(bc1, bc2)
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_BC) as g:
        g.init()
        g.bc_run([a])
        g.bc_run([b])
        assert np.array_equal(g.values(), bc1)
        state_ab = g.bc_source_state()
    _, state_b, _, _ = run_bc(row_end, src, [b])
    for x, y in zip(state_ab, state_b):
        assert np.array_equal(x, y)


def test_sources_listed_twice_count_twice_and_stats():
    row_end, src = rmat(12)
    once, _, _, st1 = run_bc(row_end, src, [5])
    twice, _, _, st2 = run_bc(row_end, src, [5, 5])
    assert np.array_equal(twice, once + once)
    assert st2["iterations"] == 2 * st1["iterations"] and st2["edges_processed"] == 2 * st1["edges_processed"]
    assert st1["loop_seconds"] > 0


def test_phase_timing_counts_sources(monkeypatch, capfd):
    # LUXB_PHASE_TIMING=2 prints the σ / δ means of every luxb_bc_run call over its sources; the BFS's own pull sweeps
    # (which PageRank's timer counts as iterations) must not enter the count
    monkeypatch.setenv("LUXB_PHASE_TIMING", "2")
    row_end, src = rmat(16)
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_BC) as g:
        g.init()
        capfd.readouterr()
        g.bc_run([0])
        assert g.trace()[1].sum() > 0  # the BFS pulled
        g.bc_run([0, 12345, 7])
        err = capfd.readouterr().err
    counts = [int(c) for c in re.findall(r"phase means over (\d+) sources:.*bc_sigma [0-9.]+ ms; bc_delta [0-9.]+ ms;", err)]
    assert counts == [1, 3], err


def test_values_are_the_scores():
    row_end, src = rmat(12)
    nv = len(row_end)
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_BC) as g:
        g.init()
        assert np.array_equal(g.values(), np.zeros(nv))
        base = np.arange(nv, dtype=np.float64) * 0.5
        g.set_values(base)
        g.bc_run([3])
        close(g.values() - base, B.scores(row_end, src, [3]))
        assert np.array_equal(g.local_values(), g.values())


def test_errors():
    row_end, src = rmat(10)
    nv = len(row_end)
    lib = L.load_library()
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_BC) as g:
        with pytest.raises(L.LuxError, match=r"\(-5\)"):   # before luxb_init
            g.bc_run([0])
        g.init()
        with pytest.raises(L.LuxError, match=r"\(-5\)"):   # no source yet
            g.bc_source_state()
        g.bc_run([1])
        before = g.values()
        with pytest.raises(L.LuxError, match=r"\(-1\).*>= nv"):
            g.bc_run([2, nv, 3])  # validated before any work: nothing is added
        assert np.array_equal(g.values(), before)
        assert lib.luxb_bc_run(g._h, None, 0) == 0 and np.array_equal(g.values(), before)
        for call in (lambda: g.iterate(1), lambda: g.run_to_convergence(), lambda: g.check()):
            with pytest.raises(L.LuxError, match=r"\(-1\).*luxb_bc_run"):
                call()
        assert lib.luxb_bc_source_state(g._h, None, None, None, C_size(nv + 1)) == -1
        assert lib.luxb_bc_source_state(g._h, None, None, None, C_size(nv)) == 0  # NULL skips every array
        assert np.array_equal(g.values(), before)
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_SSSP) as g:
        g.init()
        with pytest.raises(L.LuxError, match=r"\(-1\)"):
            g.bc_run([0])
        with pytest.raises(L.LuxError, match=r"\(-1\)"):
            g.bc_source_state()


def C_size(n):
    import ctypes
    return ctypes.c_size_t(n)


def test_apps_and_torch_op():
    import torch
    import lux_b200.torch_ops  # noqa: F401
    row_end, src = rmat(11)
    nv = len(row_end)
    close(L.betweenness(row_end, src), B.scores(row_end, src))
    S = np.array([4, 9, 4, 100], np.int64)
    t = torch.ops.luxb.betweenness(torch.from_numpy(row_end.astype(np.int64)).cuda(), torch.from_numpy(src.astype(np.int64)).cuda(),
                                   torch.from_numpy(S).cuda())
    assert t.dtype == torch.float64 and t.is_cuda and t.shape == (nv,)
    close(t.cpu().numpy(), B.scores(row_end, src, S))


def cli(*args):
    p = subprocess.run([sys.executable, os.path.join(ROOT, "apps", "lux_cli.py"), "bc"] + list(args), cwd=ROOT, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    return p.stdout


def test_cli(tmp_path):
    row_end, src = rmat(11)
    nv = len(row_end)
    path = str(tmp_path / "g.lux")
    L.write_lux(path, row_end, src)
    out = str(tmp_path / "bc.npy")
    text = cli("-file", path, "-nsrc", "16", "-seed", "5", "-out", out)
    assert re.search(r"ELAPSED TIME = \d", text) and "[Memory Setting]" not in text
    S = np.random.default_rng(5).choice(nv, 16, replace=False)
    close(np.load(out), B.scores(row_end, src, S))
    cli("-file", path, "-start", "7", "-out", out)
    close(np.load(out), B.scores(row_end, src, [7]))
    cli("-file", path, "-out", out)
    close(np.load(out), B.scores(row_end, src))


@heavy
def test_c4_rmat24():
    from test_gpu_configs import check_blocks_against_oracle_generator, scale_of
    nv, ne, seed = 1 << 24, 16 << 24, 24
    s1 = int(np.random.default_rng(24).integers(1, nv))
    with L.LuxGraph.from_rmat(scale_of(nv), nv, ne, seed, app=L.APP_BC) as g:
        row_end, src = g.local_csc()
        g.init()
        g.bc_run([0])
        lev0, sigma0, delta0 = g.bc_source_state()
        g.bc_run([s1])
        bc = g.values()
        state1 = g.bc_source_state()
    check_blocks_against_oracle_generator(scale_of(nv), nv, ne, seed, row_end, src)
    ref0 = B.run(row_end, src, [0])
    ref = B.run(row_end, src, [0, s1])
    check_state_arrays((lev0, sigma0, delta0), ref0)
    check_state_arrays(state1, ref)
    close(bc, ref["scores"])
    print("C4 BC: source 0 %d levels, source %d %d levels" % (ref0["levels"][0], s1, ref["levels"][1]))


def check_state_arrays(state, ref):
    lev, sigma, delta = state
    assert ref["sigma"].max() < 2.0 ** 53
    assert np.array_equal(lev, ref["lev"]) and np.array_equal(sigma, ref["sigma"])
    close(delta, ref["delta"])


def _run_worker(world, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mgpu_bc_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    return p.returncode, p.stdout + p.stderr


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_bc(world, gpu_count):
    if gpu_count < world:
        pytest.skip("needs %d GPUs, have %d" % (world, gpu_count))
    rc, out = _run_worker(world, 29570 + world)
    assert rc == 0 and "MGPU_BC PASS" in out, out[-4000:]
