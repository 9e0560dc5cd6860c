"""GPU parity of weighted betweenness centrality (LUXB_BC_WEIGHTED) against the CPU oracle tests/bc_weighted_oracle.c,
which tests/test_bc_weighted_oracle.py pins to networkx, scipy's Dijkstra and hand-worked graphs.  Per source: the
distances and the path counts sigma bit for bit (the oracle's sigma < 2^53 is asserted, so both are exact integers),
delta and the scores within rtol 1e-10 with exact zeros.  On the weighted forest (bc_weighted_oracle.forest) every
summation order is exact: everything bit for bit, through both split paths.  Unit weights give LUXB_BC bit for bit.
Also: the saturation chain, the weighted SSSP trace, reproducibility, error codes, the public surfaces, C4 with generator
weights and several GPUs.  LUXB_SKIP_HEAVY=1 skips C4."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import lux_b200 as L
import bc_weighted_oracle as W
import weighted_oracle as WO
from graphs import ALL_SMALL, rmat

pytestmark = pytest.mark.gpu
heavy = pytest.mark.skipif(os.environ.get("LUXB_SKIP_HEAVY") == "1", reason="LUXB_SKIP_HEAVY=1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEEP = {"chain", "two_components"}  # up to 3000 distance classes per source: sources are sampled


def close(got, want, rtol=1e-10):
    assert np.array_equal(got == 0, want == 0), "zeros differ at %s" % np.nonzero((got == 0) != (want == 0))[0][:10]
    np.testing.assert_allclose(got, want, rtol=rtol, atol=0)


def check_state(state, ref_dist, ref_sigma, ref_delta):
    dist, sigma, delta = state
    assert ref_sigma.max() < 2.0 ** 53, "the oracle's sigma is no longer an exact integer"
    assert np.array_equal(dist, ref_dist), "distances differ at %s" % np.nonzero(dist != ref_dist)[0][:10]
    assert np.array_equal(sigma, ref_sigma), "sigma differs at %s" % np.nonzero(sigma != ref_sigma)[0][:10]
    close(delta, ref_delta)


def weights(kind, ne, seed=7):
    rng = np.random.default_rng(seed)
    return (rng.integers(1, 256, ne) if kind == "w255" else rng.integers(1, 3, ne)).astype(np.int32)


def sources_for(name, nv):
    if nv <= 4096 and name not in DEEP:
        return np.arange(nv, dtype=np.uint32)
    return np.unique(np.concatenate([[0, nv - 1], np.random.default_rng(1).choice(nv, 24, replace=False)])).astype(np.uint32)


def open_bc(row_end, src, w, app=L.APP_BC_WEIGHTED, **kw):
    return L.LuxGraph.from_csc(row_end, src, w, app=app, **kw)


def per_source_parity(row_end, src, w, sources, **kw):
    """One handle, one bc_run per source: every source's state against the oracle, then the summed scores."""
    with open_bc(row_end, src, w, **kw) as g:
        g.init()
        for s in sources:
            g.bc_run([s])
            check_state(g.bc_source_state(), *W.source_state(row_end, src, w, s))
        bc = g.values()
        st = g.stats()
    close(bc, W.scores(row_end, src, w, sources))
    return st


@pytest.mark.parametrize("kind", ["w255", "w12"])
@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_small_fixtures(name, kind):
    row_end, src = ALL_SMALL[name]()
    per_source_parity(row_end, src, weights(kind, len(src)), sources_for(name, len(row_end)))


@pytest.mark.parametrize("scale", [14, 16])
def test_rmat_generator_weights(scale):
    row_end, src = rmat(scale)
    w = WO.rmat_weights(27, row_end, src)
    sources = np.random.default_rng(scale).choice(len(row_end), 8, replace=False).astype(np.uint32)
    st = per_source_parity(row_end, src, w, sources)
    assert st["iterations"] >= 8 and st["edges_processed"] > 0


def run_bc(row_end, src, w, sources, app=L.APP_BC_WEIGHTED, **kw):
    with open_bc(row_end, src, w, app=app, **kw) as g:
        g.init()
        g.bc_run(sources)
        return g.values(), g.bc_source_state(), g.trace(), g.stats()


@pytest.mark.parametrize("make", [W.small_forest, W.forest])
@pytest.mark.parametrize("config", ["default", "zero_copy"])
def test_exact_forest(make, config):
    f = make()
    ref = W.run(f["row_end"], f["src"], f["weight"], f["roots"])
    bc, (dist, sigma, delta), _, _ = run_bc(f["row_end"], f["src"], f["weight"], f["roots"], zero_copy=config == "zero_copy")
    assert np.array_equal(bc, f["scores"]) and np.array_equal(bc, ref["scores"])
    assert np.array_equal(dist, ref["dist"]) and np.array_equal(sigma, ref["sigma"]) and np.array_equal(delta, ref["delta"])


def unit_weight_pair(row_end, src, sources):
    ones = np.ones(len(src), np.int32)
    with open_bc(row_end, src, ones) as gw, L.LuxGraph.from_csc(row_end, src, app=L.APP_BC) as gu:
        gw.init()
        gu.init()
        for s in sources:
            gw.bc_run([s])
            gu.bc_run([s])
            (dw, sw, tw), (lu, su, tu) = gw.bc_source_state(), gu.bc_source_state()
            assert np.array_equal(np.where(dw == L.DIST_INF, len(row_end), dw), lu)
            assert np.array_equal(sw, su) and np.array_equal(tw, tu)
        assert np.array_equal(gw.values(), gu.values())


def test_unit_weights_are_bc_bit_for_bit_rmat15():
    row_end, src = rmat(15)
    unit_weight_pair(row_end, src, np.random.default_rng(15).choice(len(row_end), 6, replace=False).astype(np.uint32))


def test_unit_weights_are_bc_bit_for_bit_forest():
    f = W.forest()
    unit_weight_pair(f["row_end"], f["src"], f["roots"])


def test_saturation_chain():
    big = (1 << 31) - 1
    row_end, src, w = W.edges_to_csc(5, [0, 1, 2, 2], [1, 2, 3, 4], [big, big, big, 1])
    ref = W.run(row_end, src, w, [0, 1])
    bc, state, _, _ = run_bc(row_end, src, w, [0, 1])
    check_state(state, ref["dist"], ref["sigma"], ref["delta"])
    _, state0, _, _ = run_bc(row_end, src, w, [0])
    assert state0[0].tolist() == [0, big, 2 * big, L.DIST_INF, L.DIST_INF]  # 2^32 - 2 reached, 2^32 - 1 is not
    assert np.array_equal(bc, ref["scores"]) and np.all(np.isfinite(bc))


def test_trace_is_the_weighted_sssp_trace():
    row_end, src = rmat(16)
    w = WO.rmat_weights(27, row_end, src)
    for s in (0, 12345):
        _, (dist, _, _), (active, pull), _ = run_bc(row_end, src, w, [7, s])
        ref = WO.label_run(row_end, src, w, start=s)
        assert np.array_equal(dist, ref["labels"])
        assert np.array_equal(active, ref["active"]) and np.array_equal(pull, ref["pull"])
        assert pull.sum() > 0  # the pull direction took part


def test_one_rank_is_bitwise_reproducible():
    row_end, src = rmat(15)
    w = WO.rmat_weights(27, row_end, src)
    a, b = 11, 2024
    bc1, _, _, _ = run_bc(row_end, src, w, [a, b])
    bc2, _, _, _ = run_bc(row_end, src, w, [a, b])
    assert np.array_equal(bc1, bc2)
    with open_bc(row_end, src, w) as g:
        g.init()
        g.bc_run([a])
        g.bc_run([b])
        assert np.array_equal(g.values(), bc1)
        state_ab = g.bc_source_state()
    _, state_b, _, _ = run_bc(row_end, src, w, [b])
    for x, y in zip(state_ab, state_b):
        assert np.array_equal(x, y)


def test_sources_listed_twice_count_twice_and_stats():
    row_end, src = rmat(12)
    w = weights("w255", len(src))
    once, _, _, st1 = run_bc(row_end, src, w, [5])
    twice, _, _, st2 = run_bc(row_end, src, w, [5, 5])
    assert np.array_equal(twice, once + once)
    assert st2["iterations"] == 2 * st1["iterations"] and st2["edges_processed"] == 2 * st1["edges_processed"]
    assert st1["loop_seconds"] > 0


def test_phase_timing_counts_sources(monkeypatch, capfd):
    monkeypatch.setenv("LUXB_PHASE_TIMING", "2")
    row_end, src = rmat(16)
    w = WO.rmat_weights(27, row_end, src)
    with open_bc(row_end, src, w) as g:
        g.init()
        capfd.readouterr()
        g.bc_run([0])
        assert g.trace()[1].sum() > 0  # the weighted SSSP pulled
        g.bc_run([0, 12345, 7])
        err = capfd.readouterr().err
    counts = [int(c) for c in re.findall(r"phase means over (\d+) sources:.*bc_sigma [0-9.]+ ms; bc_delta [0-9.]+ ms;", err)]
    assert counts == [1, 3], err


def test_values_are_the_scores():
    row_end, src = rmat(12)
    w = weights("w255", len(src))
    nv = len(row_end)
    with open_bc(row_end, src, w) as g:
        g.init()
        assert np.array_equal(g.values(), np.zeros(nv))
        base = np.arange(nv, dtype=np.float64) * 0.5
        g.set_values(base)
        g.bc_run([3])
        close(g.values() - base, W.scores(row_end, src, w, [3]))
        assert np.array_equal(g.local_values(), g.values())


@pytest.mark.parametrize("bad", [0, -3])
def test_weights_below_one_fail_the_open(bad):
    row_end, src = rmat(10)
    w = weights("w255", len(src))
    w[[5, 77, 300]] = bad
    with pytest.raises(L.LuxError, match=r"\(-1\).*3 edge weights .* < 1 .*w >= 1"):
        open_bc(row_end, src, w)
    w[[5, 77, 300]] = 1
    open_bc(row_end, src, w).close()


def test_errors():
    row_end, src = rmat(10)
    nv = len(row_end)
    lib = L.load_library()
    with pytest.raises(L.LuxError, match=r"\(-1\).*weighted betweenness centrality needs edge weights"):
        open_bc(row_end, src, None)
    w = weights("w255", len(src))
    with open_bc(row_end, src, w) as g:
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
        assert lib.luxb_bc_source_state(g._h, None, None, None, ctypes.c_size_t(nv + 1)) == -1
        assert np.array_equal(g.values(), before)


def test_apps_and_torch_op():
    import torch
    import lux_b200.torch_ops  # noqa: F401
    row_end, src = rmat(11)
    nv = len(row_end)
    w = weights("w255", len(src))
    close(L.betweenness(row_end, src, weight=w), W.scores(row_end, src, w))
    S = np.array([4, 9, 4, 100], np.int64)
    t = torch.ops.luxb.betweenness_weighted(torch.from_numpy(row_end.astype(np.int64)).cuda(),
                                            torch.from_numpy(src.astype(np.int64)).cuda(), torch.from_numpy(w).cuda(),
                                            torch.from_numpy(S).cuda())
    assert t.dtype == torch.float64 and t.is_cuda and t.shape == (nv,)
    close(t.cpu().numpy(), W.scores(row_end, src, w, S))


def cli(*args):
    p = subprocess.run([sys.executable, os.path.join(ROOT, "apps", "lux_cli.py"), "bc"] + list(args), cwd=ROOT, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    return p.stdout


def test_cli(tmp_path):
    row_end, src = rmat(11)
    nv = len(row_end)
    w = weights("w255", len(src))
    path = str(tmp_path / "w.lux")
    L.write_lux(path, row_end, src, w)
    out = str(tmp_path / "bc.npy")
    text = cli("-weighted", "-file", path, "-nsrc", "16", "-seed", "5", "-out", out)
    assert re.search(r"ELAPSED TIME = \d", text) and "[Memory Setting]" not in text
    S = np.random.default_rng(5).choice(nv, 16, replace=False)
    close(np.load(out), W.scores(row_end, src, w, S))
    cli("-weighted", "-file", path, "-start", "7", "-out", out)
    close(np.load(out), W.scores(row_end, src, w, [7]))
    cli("-weighted", "-file", path, "-out", out)
    close(np.load(out), W.scores(row_end, src, w))


@heavy
def test_c4_weighted_rmat24():
    from test_gpu_configs import check_blocks_against_oracle_generator, scale_of
    nv, ne, seed = 1 << 24, 16 << 24, 24
    s1 = int(np.random.default_rng(24).integers(1, nv))
    with L.LuxGraph.from_rmat(scale_of(nv), nv, ne, seed, app=L.APP_BC_WEIGHTED) as g:
        row_end, src, w = g.local_csc(weighted=True)
        g.init()
        g.bc_run([0])
        state0 = g.bc_source_state()
        g.bc_run([s1])
        bc = g.values()
        state1 = g.bc_source_state()
    check_blocks_against_oracle_generator(scale_of(nv), nv, ne, seed, row_end, src)
    assert np.array_equal(w, WO.rmat_weights(seed, row_end, src))
    ref0 = W.run(row_end, src, w, [0])
    ref1 = W.run(row_end, src, w, [s1])
    check_state(state0, ref0["dist"], ref0["sigma"], ref0["delta"])
    check_state(state1, ref1["dist"], ref1["sigma"], ref1["delta"])
    scores = np.zeros(nv)  # the oracle's accumulation, source by source
    for s, r in ((0, ref0), (s1, ref1)):
        mask = np.arange(nv) != s
        scores[mask] += r["delta"][mask]
    close(bc, scores)
    print("C4 weighted BC: source 0 %d distance classes, source %d %d" % (ref0["classes"][0], s1, ref1["classes"][0]))


def _run_worker(world, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mgpu_bc_weighted_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    return p.returncode, p.stdout + p.stderr


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_bc_weighted(world, gpu_count):
    if gpu_count < world:
        pytest.skip("needs %d GPUs, have %d" % (world, gpu_count))
    rc, out = _run_worker(world, 29590 + world)
    assert rc == 0 and "MGPU_BC_WEIGHTED PASS" in out, out[-4000:]
