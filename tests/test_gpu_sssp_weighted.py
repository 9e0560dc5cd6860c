"""GPU parity of weighted SSSP (LUXB_SSSP_WEIGHTED) against the weighted CPU oracle, which tests/
test_sssp_weighted_oracle.py pins to scipy's Dijkstra: bit-exact labels, the same iteration count, the same
per-iteration global active counts and pull/push decisions, and luxb_check == 0.  The push kernels (inline and
hub-segment), the merge-path pull sweep with its weight ring in every shape, zero-copy edges, the device generators,
the check predicate, the public surfaces and C4 as BASELINE states it (weighted RMAT-24, start 0).
LUXB_SKIP_HEAVY=1 skips C4 (a minute of host work for the oracle)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
import lux_b200 as L
import weighted_oracle as W
from graphs import ALL_SMALL, rmat, star
from test_gpu_configs import check_blocks_against_oracle_generator, scale_of

pytestmark = pytest.mark.gpu
heavy = pytest.mark.skipif(os.environ.get("LUXB_SKIP_HEAVY") == "1", reason="LUXB_SKIP_HEAVY=1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INF = 0xFFFFFFFF


def random_weights(ne, seed, hi=20):
    return np.random.default_rng(seed).integers(0, hi, ne).astype(np.int32)


def compare(row_end, src, w, start=0, **kw):
    ref = W.label_run(row_end, src, w, P=1, start=start)
    with L.LuxGraph.from_csc(row_end, src, w, app=L.APP_SSSP_WEIGHTED, start=start, **kw) as g:
        g.init()
        it = g.run_to_convergence()
        lab = g.values()
        bad = g.check()
        active, pull = g.trace()
        st = g.stats()
    assert np.array_equal(lab, ref["labels"]), "labels differ at %s" % np.nonzero(lab != ref["labels"])[0][:10]
    assert bad == 0
    assert it == ref["iters"]
    assert np.array_equal(active, ref["active"]) and np.array_equal(pull, ref["pull"])
    return ref, st


@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_small_graphs_two_starts(name):
    row_end, src = ALL_SMALL[name]()
    w = random_weights(len(src), 7)
    for start in (0, len(row_end) - 1):
        compare(row_end, src, w, start=start)


def test_zero_weights():
    row_end, src = rmat(14)
    ref, _ = compare(row_end, src, np.zeros(len(src), np.int32))
    assert set(np.unique(ref["labels"]).tolist()) <= {0, INF}


def test_saturating_weights():
    # a chain whose third hop would pass 2^32 - 1: INF, not a wrapped small distance
    row_end, src = O.edges_to_csc(4, [0, 1, 2], [1, 2, 3])
    ref, _ = compare(row_end, src, np.array([2**31 - 1, 2**31 - 1, 5], np.int32))
    assert ref["labels"].tolist() == [0, 2**31 - 1, 2**32 - 2, INF]
    # a graph where many paths saturate, through both directions
    row_end, src = rmat(14)
    w = (np.int64(2**30) + random_weights(len(src), 2, hi=1 << 20)).astype(np.int32)
    ref, _ = compare(row_end, src, w)
    reachable = O.label_run(O.APP_SSSP, row_end, src, P=1, start=0)["labels"] < len(row_end)
    assert (reachable & (ref["labels"] == INF)).sum() > 0 and ref["pull"].sum() > 0  # saturated, not merely unreachable


def test_push_big_kernel_star_source():
    # vertex 0 has 9999 out-edges (> kPushBigDegree = 2048): the first push step runs through push_big_kernel
    row_end, src = star(10000, both=True)
    compare(row_end, src, random_weights(len(src), 3, hi=1000), start=0)
    # the same with unique weights so that a neighbouring edge's weight gives a different answer
    w = np.random.default_rng(4).permutation(len(src)).astype(np.int32)
    compare(row_end, src, w, start=0)


def test_unit_weights_equal_hop_counts():
    row_end, src = rmat(16)
    nv = len(row_end)
    hop = L.sssp(row_end, src, start=0, check=True)
    out = L.sssp(row_end, src, start=0, check=True, weight=np.ones(len(src), np.int32))
    mapped = np.where(hop["labels"] == nv, np.uint32(INF), hop["labels"])
    assert np.array_equal(out["labels"], mapped) and out["mistakes"] == 0
    assert out["iters"] == hop["iters"]
    assert np.array_equal(out["trace"][0], hop["trace"][0]) and np.array_equal(out["trace"][1], hop["trace"][1])


@pytest.mark.parametrize("shape", [0, 1, 2])
def test_every_pull_shape(shape, monkeypatch):
    monkeypatch.setenv("LUXB_PULL_SHAPE", str(shape))
    row_end, src = rmat(15)
    _, st = compare(row_end, src, random_weights(len(src), 5, hi=100))
    assert st["pull_iterations"] > 0


def test_zero_copy_edges():
    row_end, src = rmat(15)
    _, st = compare(row_end, src, random_weights(len(src), 6, hi=100), zero_copy=True)
    assert st["pull_iterations"] > 0


def test_seg_sweep_settings_have_no_effect(monkeypatch):
    # weighted SSSP pulls through the merge path only: forcing the flagged sweeps changes nothing
    monkeypatch.setenv("LUXB_SB", "1")
    monkeypatch.setenv("LUXB_SB_BS", "64")
    monkeypatch.setenv("LUXB_SB_MIN_INDEG", "4")
    row_end, src = rmat(14)
    compare(row_end, src, random_weights(len(src), 8, hi=50))


def test_device_generated_rmat18():
    scale, seed = 18, 24
    nv, ne = 1 << scale, 16 << scale
    with L.LuxGraph.from_rmat(scale, nv, ne, seed, app=L.APP_SSSP_WEIGHTED, start=0) as g:
        row_end, src, w = g.local_csc(weighted=True)
        g.init()
        it = g.run_to_convergence()
        lab = g.values()
        assert g.check() == 0
        active, pull = g.trace()
    re_o, src_o = O.gen_rmat_csc(scale, nv, ne, seed)
    w_o = W.rmat_weights(seed, re_o, src_o)
    assert np.array_equal(row_end, re_o) and np.array_equal(src, src_o) and np.array_equal(w, w_o)
    ref = W.label_run(re_o, src_o, w_o, P=1, start=0)
    assert it == ref["iters"] and np.array_equal(lab, ref["labels"])
    assert np.array_equal(active, ref["active"]) and np.array_equal(pull, ref["pull"])


def test_bipartite():
    users, items, ratings, seed = 3000, 300, 60000, 5
    re_b, src_b, w_b = O.gen_bipartite_csc(users, items, ratings, seed)
    with L.LuxGraph.from_bipartite(users, items, ratings, seed, app=L.APP_SSSP_WEIGHTED, start=1) as g:
        row_end, src, w = g.local_csc(weighted=True)
        g.init()
        it = g.run_to_convergence()
        lab = g.values()
        assert g.check() == 0
    assert np.array_equal(src, src_b) and np.array_equal(w, w_b)
    ref = W.label_run(re_b, src_b, w_b, P=1, start=1)
    assert it == ref["iters"] and np.array_equal(lab, ref["labels"])


def test_check_counts_mistakes_like_the_oracle():
    row_end, src = rmat(14)
    nv = len(row_end)
    w = random_weights(len(src), 9, hi=30)
    ref = W.label_run(row_end, src, w, P=1, start=0)["labels"]
    rng = np.random.default_rng(11)
    with L.LuxGraph.from_csc(row_end, src, w, app=L.APP_SSSP_WEIGHTED, start=0) as g:
        g.init()
        g.run_to_convergence()
        assert g.check() == 0
        for k in (1, 7, 300):
            bad = ref.copy()
            idx = rng.choice(nv, k, replace=False)
            bad[idx] = np.where(bad[idx] == INF, rng.integers(0, 50, k), bad[idx].astype(np.int64) + rng.integers(31, 90, k)).astype(np.uint32)
            want = W.label_check(row_end, src, w, bad)
            g.set_values(bad)
            got = g.check()
            assert got == want, (k, got, want)
            if k >= 7:
                assert want > 0
        g.set_values(ref)
        assert g.check() == 0


def test_negative_weight_fails_the_open():
    row_end, src = rmat(10)
    w = np.ones(len(src), np.int32)
    w[len(w) // 2] = -1
    with pytest.raises(L.LuxError, match="negative"):
        L.LuxGraph.from_csc(row_end, src, w, app=L.APP_SSSP_WEIGHTED, start=0)
    with pytest.raises(L.LuxError):
        L.LuxGraph.from_csc(row_end, src, None, app=L.APP_SSSP_WEIGHTED, start=0)


def test_unweighted_sssp_ignores_weights():
    row_end, src = rmat(14)
    w = random_weights(len(src), 1, hi=100)
    ref = O.label_run(O.APP_SSSP, row_end, src, P=1, start=0)
    with L.LuxGraph.from_csc(row_end, src, w, app=L.APP_SSSP, start=0) as g:
        g.init()
        it = g.run_to_convergence()
        assert np.array_equal(g.values(), ref["labels"]) and it == ref["iters"] and g.check() == 0


def test_torch_op_and_apps_entry():
    import torch
    import lux_b200.torch_ops  # noqa: F401
    row_end, src = rmat(12)
    w = random_weights(len(src), 12, hi=40)
    ref = W.label_run(row_end, src, w, P=1, start=3)
    out = L.sssp(row_end, src, start=3, check=True, weight=w)
    assert np.array_equal(out["labels"], ref["labels"]) and out["mistakes"] == 0
    t = torch.ops.luxb.sssp_weighted(torch.from_numpy(row_end.astype(np.int64)).cuda(), torch.from_numpy(src.astype(np.int64)).cuda(),
                                     torch.from_numpy(w).cuda(), 3)
    assert t.dtype == torch.int64 and t.is_cuda
    assert np.array_equal(t.cpu().numpy(), ref["labels"].astype(np.int64))


def test_cli_weighted_check_out(tmp_path):
    row_end, src = rmat(12)
    w = random_weights(len(src), 13, hi=40)
    path = str(tmp_path / "w.lux")
    L.write_lux(path, row_end, src, w)
    out = str(tmp_path / "d.npy")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "apps", "lux_cli.py"), "sssp", "-weighted", "-file", path, "-start", "5",
                        "-check", "-out", out], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    assert "[PASS] Check task" in p.stdout and "ELAPSED TIME" in p.stdout and "[Memory Setting]" in p.stdout
    ref = W.label_run(row_end, src, w, P=1, start=5)
    assert np.array_equal(np.load(out), ref["labels"])


@heavy
def test_c4_weighted_sssp_rmat24_start0():
    nv, ne, seed = 1 << 24, 16 << 24, 24
    with L.LuxGraph.from_rmat(scale_of(nv), nv, ne, seed, app=L.APP_SSSP_WEIGHTED, start=0) as g:
        row_end, src, w = g.local_csc(weighted=True)
        g.init()
        it = g.run_to_convergence()
        lab = g.values()
        bad = g.check()
        active, pull = g.trace()
    check_blocks_against_oracle_generator(scale_of(nv), nv, ne, seed, row_end, src)
    w_o = W.rmat_weights(seed, row_end, src)
    assert np.array_equal(w, w_o), "device weights differ from the oracle generator"
    del w
    ref = W.label_run(row_end, src, w_o, P=1, start=0)
    assert np.array_equal(lab, ref["labels"])
    assert bad == 0 and W.label_check(row_end, src, w_o, lab) == 0
    assert it == ref["iters"]
    assert np.array_equal(active, ref["active"]) and np.array_equal(pull, ref["pull"])
    print("C4 weighted: %d iterations, %d pull" % (it, int(pull.sum())))


def _run_worker(world, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mgpu_sssp_weighted_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    return p.returncode, p.stdout + p.stderr


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_weighted_sssp(world, gpu_count):
    if gpu_count < world:
        pytest.skip("needs %d GPUs, have %d" % (world, gpu_count))
    rc, out = _run_worker(world, 29560 + world)
    assert rc == 0 and "MGPU_SSSP_W PASS" in out, out[-4000:]
