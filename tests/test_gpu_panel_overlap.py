"""The concurrent split sweep (api.cu: sweep_seg) on the device: the panel kernel on LUXB_PANEL_SMS SMs while the
cold-hub and main kernels run beside it on a second stream, then a join launch of the main kernel on the panel's SMs.

Every stage is still claimed exactly once and the fix-ups are unchanged, so the results must be bit for bit those of
the serial schedule (LUXB_PANEL_SMS=0) and, on exact inputs, of the oracle (the method of test_gpu_exact.py).  The
concurrent schedule launches the main kernel twice per sweep, so it shows as one more kernel launch per sweep.

Covered: exact inputs through the forced split and the forced cold-hub stream at RMAT-22 with 1, 8, the default and
all but one SM for the panel; 20 ordinary iterations against the serial schedule; CC and SSSP through the split; a
panel SM count of at least the SM count falling back to the serial schedule; a handle opened and closed 50 times."""
import functools

import numpy as np
import pytest
import torch

import oracle as O
import lux_b200 as L
from graphs import rmat, symmetrize
from test_gpu_exact import assert_bit_equal, exact_steps, set_env

pytestmark = pytest.mark.gpu

SPLIT = dict(LUXB_SB=1, LUXB_SB_BS=512, LUXB_SB_BLOCKS=8, LUXB_SB_MIN_INDEG=16)
# at RMAT-22 the whole graph fits the default hot set: a smaller one leaves cold sources for the cold-hub stream
COLD = dict(LUXB_SB=1, LUXB_CS=1, LUXB_HOT_MB=4, LUXB_CS_SEG_MB=2)


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@functools.lru_cache(maxsize=None)
def graph(name):
    if name == "rmat16_sym":
        return symmetrize(*rmat(16, ef=8))
    if name == "rmat22":
        return O.gen_rmat_csc(22, 1 << 22, 16 << 22, 27)
    return rmat(int(name[len("rmat"):]))


def pagerank_run(name, env, monkeypatch, iters):
    """values and kernel launches of `iters` iterations from the initial values"""
    monkeypatch.delenv("LUXB_PANEL_SMS", raising=False)
    set_env(monkeypatch, env)
    row_end, src = graph(name)
    with L.LuxGraph.from_csc(row_end, src) as g:
        g.init()
        st = g.stats()
        k0 = g.stats()["kernel_launches"]
        g.iterate(iters)
        return g.values(), g.stats()["kernel_launches"] - k0, st


@pytest.mark.parametrize("panel_sms", ["1", "8", "default", "all_but_one"])
def test_exact_rmat22_split_and_cold_hub(panel_sms, monkeypatch):
    env = dict(COLD)
    if panel_sms != "default":
        env["LUXB_PANEL_SMS"] = num_sms() - 1 if panel_sms == "all_but_one" else int(panel_sms)
    set_env(monkeypatch, env)
    row_end, src = graph("rmat22")
    with L.LuxGraph.from_csc(row_end, src) as g:
        g.init()
        st = g.stats()
        assert st["panel_edges"] > 0 and st["cold_hub_edges"] > 0, st
        exact_steps(g, row_end, src, "rmat22 LUXB_PANEL_SMS=%s" % panel_sms, rounds=2)


def test_values_match_serial_schedule_20_iterations(monkeypatch):
    serial, n_serial, _ = pagerank_run("rmat22", dict(COLD, LUXB_PANEL_SMS=0), monkeypatch, 20)
    beside, n_beside, st = pagerank_run("rmat22", COLD, monkeypatch, 20)
    assert st["panel_edges"] > 0 and st["cold_hub_edges"] > 0, st
    assert n_beside == n_serial + 20  # the join launch of the main kernel, once per sweep
    assert_bit_equal(beside, serial, "rmat22, 20 iterations, default vs LUXB_PANEL_SMS=0")


@pytest.mark.parametrize("over", [0, 5])
def test_panel_sms_at_least_the_sm_count_is_serial(over, monkeypatch):
    serial, n_serial, _ = pagerank_run("rmat17", dict(SPLIT, LUXB_PANEL_SMS=0), monkeypatch, 3)
    got, n_got, st = pagerank_run("rmat17", dict(SPLIT, LUXB_PANEL_SMS=num_sms() + over), monkeypatch, 3)
    assert st["panel_edges"] > 0, st
    assert n_got == n_serial
    assert_bit_equal(got, serial, "LUXB_PANEL_SMS = SMs + %d" % over)


def label_run(app, name, env, monkeypatch):
    monkeypatch.delenv("LUXB_PANEL_SMS", raising=False)
    set_env(monkeypatch, env)
    row_end, src = graph(name)
    with L.LuxGraph.from_csc(row_end, src, app=app, start=0) as g:
        g.init()
        st = g.stats()
        it = g.run_to_convergence()
        return g.values(), it, g.trace(), g.stats()["kernel_launches"], st


@pytest.mark.parametrize("app_name", ["cc", "sssp"])
def test_labels_through_the_concurrent_split(app_name, monkeypatch):
    app, oapp, name = (L.APP_CC, O.APP_CC, "rmat16_sym") if app_name == "cc" else (L.APP_SSSP, O.APP_SSSP, "rmat16")
    row_end, src = graph(name)
    ref = O.label_run(oapp, row_end, src, P=1, start=0)
    _, _, _, n_serial, _ = label_run(app, name, dict(SPLIT, LUXB_PANEL_SMS=0), monkeypatch)
    lab, it, (active, pull), n_beside, st = label_run(app, name, SPLIT, monkeypatch)
    assert st["panel_edges"] > 0, st
    assert pull.any() and n_beside > n_serial  # join launches: the pull sweeps ran concurrently
    assert np.array_equal(lab, ref["labels"]) and it == ref["iters"]
    assert np.array_equal(active, ref["active"]) and np.array_equal(pull, ref["pull"])


def test_reopen_50_times(monkeypatch):
    """the side stream, its events and its L2 window are released at close: 50 handles in a row, the same values each time"""
    set_env(monkeypatch, SPLIT)
    row_end, src = graph("rmat16")
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    first = None
    for i in range(50):
        with L.LuxGraph.from_csc(row_end, src) as g:
            g.init()
            g.iterate(2)
            x = g.values()
        if first is None:
            first = x
        assert_bit_equal(x, first, "handle %d" % i)
    free1 = torch.cuda.mem_get_info()[0]
    assert free1 >= free0 - (64 << 20), (free0, free1)
