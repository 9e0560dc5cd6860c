"""GPU parity of triangle counting (LUXB_TC) against the CPU oracle tests/tc_oracle.c, which tests/test_tc_oracle.py pins
to networkx, scipy and closed forms.  Integers only, so everything is bit for bit: t against the oracle, sum(t) == 3 T,
stats.edges_processed == m per run.  Exact families need no oracle: K_2048 under storage noise (every vertex ties in
degree, so the id tie-break orders everything), a wheel whose hub is the w of every triangle, K_{1000,1000} (heavy
probing, no triangle), and a graph whose longest out-lists exceed the shared-memory budget kTcSharedList.  Also the
configurations, repeat runs, error codes, the public surfaces, C4 at full size and several GPUs.  LUXB_SKIP_HEAVY=1 skips
C4."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import lux_b200 as L
import tc_oracle as T
from graphs import ALL_SMALL, rmat

pytestmark = pytest.mark.gpu
heavy = pytest.mark.skipif(os.environ.get("LUXB_SKIP_HEAVY") == "1", reason="LUXB_SKIP_HEAVY=1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUDGET = 1024  # kTcSharedList (tc.cuh): longest out-list the grouped kernel stages whole


def run_tc(row_end, src, runs=1, **kw):
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_TC, **kw) as g:
        g.init()
        totals = [g.tc_run() for _ in range(runs)]
        return totals, g.values(), g.stats()


def check(row_end, src, want_t=None, **kw):
    ref = T.run(row_end, src)
    if want_t is not None:
        assert np.array_equal(ref["t"], want_t)
    (total,), t, st = run_tc(row_end, src, **kw)
    assert t.dtype == np.uint64
    assert np.array_equal(t, ref["t"]), "t differs at %s" % np.nonzero(t != ref["t"])[0][:10]
    assert total == ref["total"] and 3 * total == int(t.sum())
    assert st["edges_processed"] == ref["m"] and st["iterations"] == 1
    return ref


@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_small_fixtures(name):
    check(*ALL_SMALL[name]())


@pytest.mark.parametrize("scale", [10, 12, 14, 16, 18])
def test_rmat(scale):
    ref = check(*rmat(scale))
    assert ref["total"] > 0


@pytest.mark.parametrize("kind", T.VARIANTS)
def test_k2048_noise(kind):
    n = 2048
    row_end, src, t = T.complete(n)
    check(*T.variant(row_end, src, kind, seed=3), want_t=t)


def test_k2048_plain():
    check(*T.complete(2048))


def test_wheel_hub_contention():
    row_end, src, t = T.wheel(1 << 17)
    check(row_end, src, want_t=t)


def test_complete_bipartite():
    row_end, src, t = T.complete_bipartite(1000, 1000)
    ref = check(row_end, src, want_t=t)
    assert ref["total"] == 0 and ref["m"] == 10 ** 6


@pytest.mark.parametrize("H", [1, 37, (BUDGET + 4) // 2])
def test_out_lists_over_budget(H):
    row_end, src, t = T.over_budget(BUDGET, H)
    ref = check(row_end, src, want_t=t)
    assert ref["total"] == H * (BUDGET + 9) and ref["max_out"] == BUDGET + 4
    check(*T.variant(row_end, src, "both"), want_t=t)


def test_windmill():
    row_end, src, t = T.windmill(50000)
    check(row_end, src, want_t=t)


@pytest.mark.parametrize("config", ["zero_copy", "balanced"])
def test_configurations(config):
    row_end, src = rmat(15)
    ref = check(row_end, src, zero_copy=config == "zero_copy", balanced=config == "balanced")
    assert ref["total"] > 0


def test_rmat_generated_on_device():
    with L.LuxGraph.from_rmat(15, 1 << 15, 16 << 15, 11, app=L.APP_TC) as g:
        row_end, src = g.local_csc()
        g.init()
        total = g.tc_run()
        t = g.values()
        assert np.array_equal(g.local_values(), t)
    ref = T.run(row_end, src)
    assert total == ref["total"] and np.array_equal(t, ref["t"])


def test_repeat_runs_and_values():
    row_end, src = rmat(14)
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_TC) as g:
        g.init()
        assert not g.values().any()  # zeros before the first run
        a = g.tc_run()
        ta = g.values()
        b = g.tc_run()
        tb = g.values()
        st = g.stats()
    ref = T.run(row_end, src)
    assert a == b == ref["total"] and np.array_equal(ta, tb) and np.array_equal(ta, ref["t"])
    assert st["iterations"] == 2 and st["edges_processed"] == 2 * ref["m"] and st["loop_seconds"] > 0


def test_weighted_csc_accepted():
    row_end, src = rmat(12)
    w = np.arange(len(src), dtype=np.int32) % 7 - 3
    (total,), t, _ = run_tc(row_end, src, weight=w)
    ref = T.run(row_end, src)
    assert total == ref["total"] and np.array_equal(t, ref["t"])


def test_errors():
    row_end, src = rmat(10)
    nv = len(row_end)
    lib = L.load_library()
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_TC) as g:
        with pytest.raises(L.LuxError, match=r"\(-5\)"):   # before luxb_init
            g.tc_run()
        g.init()
        g.tc_run()
        before = g.values()
        calls = (lambda: g.iterate(1), lambda: g.run_to_convergence(), lambda: g.check(),
                 lambda: g.set_values(np.zeros(nv, np.uint64)), lambda: g.set_local_values(np.zeros(nv, np.uint64)))
        for call in calls:
            with pytest.raises(L.LuxError, match=r"\(-1\).*luxb_tc_run"):
                call()
        with pytest.raises(L.LuxError, match=r"\(-1\)"):
            g.bc_run([0])
        assert np.array_equal(g.values(), before)
        assert lib.luxb_tc_run(g._h, None) == 0  # the total is optional
    with L.LuxGraph.from_csc(row_end, src, app=L.APP_BC) as g:
        g.init()
        with pytest.raises(L.LuxError, match=r"\(-1\)"):
            g.tc_run()


def test_apps_and_torch_op():
    import torch
    import lux_b200.torch_ops  # noqa: F401
    row_end, src = rmat(11)
    ref = T.run(row_end, src)
    out = L.triangles(row_end, src)
    assert out["total"] == ref["total"] and np.array_equal(out["per_vertex"], ref["t"])
    t = torch.ops.luxb.triangles(torch.from_numpy(row_end.astype(np.int64)).cuda(), torch.from_numpy(src.astype(np.int64)).cuda())
    assert t.dtype == torch.int64 and t.is_cuda and t.shape == (len(row_end),)
    assert np.array_equal(t.cpu().numpy(), ref["t"].astype(np.int64))


def test_cli(tmp_path):
    row_end, src = rmat(11)
    path = str(tmp_path / "g.lux")
    L.write_lux(path, row_end, src)
    out = str(tmp_path / "t.npy")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "apps", "lux_cli.py"), "tc", "-file", path, "-out", out], cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    ref = T.run(row_end, src)
    assert re.search(r"ELAPSED TIME = \d", p.stdout) and "[Memory Setting]" not in p.stdout
    assert re.search(r"^TRIANGLES = %d$" % ref["total"], p.stdout, re.M)
    t = np.load(out)
    assert t.dtype == np.uint64 and np.array_equal(t, ref["t"])


@heavy
def test_c4_rmat24():
    from test_gpu_configs import check_blocks_against_oracle_generator, scale_of
    nv, ne, seed = 1 << 24, 16 << 24, 24
    with L.LuxGraph.from_rmat(scale_of(nv), nv, ne, seed, app=L.APP_TC) as g:
        row_end, src = g.local_csc()
        g.init()
        total = g.tc_run()
        t = g.values()
        st = g.stats()
    check_blocks_against_oracle_generator(scale_of(nv), nv, ne, seed, row_end, src)
    ref = T.run(row_end, src)
    assert total == ref["total"] and np.array_equal(t, ref["t"]) and st["edges_processed"] == ref["m"]
    print("C4 TC: T = %d, m = %d, max out-degree %d, probes %d" % (total, ref["m"], ref["max_out"], ref["probes"]))


def _run_worker(world, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mgpu_tc_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    return p.returncode, p.stdout + p.stderr


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_tc(world, gpu_count):
    if gpu_count < world:
        pytest.skip("needs %d GPUs, have %d" % (world, gpu_count))
    rc, out = _run_worker(world, 29610 + world)
    assert rc == 0 and "MGPU_TC PASS" in out, out[-4000:]
