"""Compact (group, hub) slots of the source-blocked split, on the device, held to the oracle bit for bit.

The panel and cold-hub streams number only the (source group, hub) pairs that have edges, in the order they close them
(panel.cuh); the combine finds a hub's partials through the slot bitmap.  A pair without edges used to add the
program's identity, which is exact, so every result here must equal the oracle exactly (np.array_equal on the bits):
one set_values + iterate(1) from integer inputs on which every summation order is exact (tests/graphs.py), as in
tests/test_gpu_exact.py.

Covered: the forced split in all six panel shapes with the tiers on and off and with the cold-hub stream forced; tiers
whose slots are mostly empty (a small LUXB_SB_SLOT_EDGES); source blocks without a single edge into a hub; hubs whose
edges all stay in the main stream; CC and SSSP through the panel with the tiers forced."""
import functools

import numpy as np
import pytest

import oracle as O
import lux_b200 as L
from graphs import exact_pr_inputs, in_degrees, rmat, symmetrize

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def graph(name):
    if name == "rmat16_sym":
        return symmetrize(*rmat(16, ef=8))
    if name == "empty_blocks":
        return empty_blocks_graph()
    return rmat(int(name[len("rmat"):]))


def empty_blocks_graph():
    """64 sources of out-degree 20 into non-hubs (the hottest: whole source blocks without a hub edge), 64 sources of
    out-degree 10 into ten hubs, and a hub fed only by 40 sources of out-degree 1 (cold: its edges stay in the main
    stream)."""
    n = 4096
    es, ed = [], []
    for i, s in enumerate(range(64, 128)):
        for k in range(20):
            es.append(s)
            ed.append(200 + (i * 20 + k) % 1500)
    for s in range(64):
        for hub in range(2000, 2010):
            es.append(s)
            ed.append(hub)
    for s in range(3000, 3040):
        es.append(s)
        ed.append(2100)
    return O.edges_to_csc(n, np.array(es), np.array(ed))


def set_env(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))


def exact_steps(name, **kw):
    row_end, src = graph(name)
    nv = len(row_end)
    deg = O.out_degree(nv, src)
    max_in = int(in_degrees(row_end).max())
    with L.LuxGraph.from_csc(row_end, src, **kw) as g:
        g.init()
        st = g.stats()
        for i, x in enumerate(exact_pr_inputs(nv, max_in)):
            g.set_values(x)
            g.iterate(1)
            got = g.values()
            ref = O.pagerank_iter(row_end, src, deg, x)
            assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), \
                "%s input %d: %d values differ" % (name, i, np.count_nonzero(got.view(np.uint32) != ref.view(np.uint32)))
    return st


SPLIT = dict(LUXB_SB=1, LUXB_SB_BS=512, LUXB_SB_BLOCKS=8, LUXB_SB_MIN_INDEG=16)


@pytest.mark.parametrize("tiers", [0, 1])
@pytest.mark.parametrize("panel_shape", range(6))
def test_forced_split_every_panel_shape(panel_shape, tiers, monkeypatch):
    set_env(monkeypatch, dict(SPLIT, LUXB_SB_TIER=tiers, LUXB_SEG_PANEL_SHAPE=panel_shape))
    st = exact_steps("rmat17")
    assert st["panel_edges"] > 0
    assert (st["tier_blocks"] > 0) == bool(tiers), st


@pytest.mark.parametrize("tiers", [0, 1])
def test_cold_hub_stream_forced(tiers, monkeypatch):
    set_env(monkeypatch, dict(SPLIT, LUXB_SB_TIER=tiers, LUXB_CS=1, LUXB_CS_SEG_MB=0.02, LUXB_HOT_MB=0.04))
    st = exact_steps("rmat16")
    assert st["cold_hub_edges"] > 0 and st["cold_hub_segments"] > 1, st


def test_tiers_with_mostly_empty_slots(monkeypatch):
    # K = 0.001 expected edges per slot keeps nearly every hub in every tier block
    set_env(monkeypatch, dict(SPLIT, LUXB_SB_BLOCKS=2, LUXB_SB_TIER=1, LUXB_SB_SLOT_EDGES=0.001))
    st = exact_steps("rmat17")
    assert st["tier_slots"] > 2 * st["tier_edges"], st  # a slot holds >= 1 edge: most tier (block, hub) pairs have none


@pytest.mark.parametrize("cs", [0, 1])
def test_blocks_without_hub_edges_and_main_only_hubs(cs, monkeypatch):
    set_env(monkeypatch, dict(LUXB_SB=1, LUXB_SB_BS=16, LUXB_SB_BLOCKS=48, LUXB_SB_MIN_INDEG=32, LUXB_SB_TIER=0, LUXB_CS=cs,
                              LUXB_HOT_MB=128 * 4e-6))
    st = exact_steps("empty_blocks")
    assert st["panel_edges"] > 0 and st["panel_blocks"] >= 5, st


@pytest.mark.parametrize("app_name", ["cc", "sssp"])
def test_labels_through_the_tiers(app_name, monkeypatch):
    set_env(monkeypatch, dict(SPLIT, LUXB_SB_TIER=1, LUXB_SB_SLOT_EDGES=0.01))
    app, oapp, name = (L.APP_CC, O.APP_CC, "rmat16_sym") if app_name == "cc" else (L.APP_SSSP, O.APP_SSSP, "rmat16")
    row_end, src = graph(name)
    with L.LuxGraph.from_csc(row_end, src, app=app, start=0) as g:
        g.init()
        st = g.stats()
        it = g.run_to_convergence()
        lab = g.values()
        active, pull = g.trace()
    ref = O.label_run(oapp, row_end, src, P=1, start=0)
    assert st["panel_edges"] > 0 and st["tier_blocks"] > 0, st
    assert pull.any()
    assert np.array_equal(lab, ref["labels"]) and it == ref["iters"]
    assert np.array_equal(active, ref["active"]) and np.array_equal(pull, ref["pull"])
