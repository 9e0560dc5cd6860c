"""GPU parity of the PageRank sweep variants against the CPU oracle, 1e-6 relative:
  * the flagged segmented-scan sweep (seg.cuh) in all its shapes — the default for every PageRank test;
  * its source-blocked split (panel.cuh: hub destinations x hot source blocks gathered from shared memory, the rest
    through L1, fp64 combine).  The split is normally enabled only on large partitions; LUXB_SB=1 with small blocks /
    thresholds forces it on small graphs so that every code path (many blocks, padding, hubs spanning pieces in both
    streams, (block, hub) pairs without edges, hubs whose edges all moved to the panel) is exercised;
  * the merge-path tiles of pull.cuh (LUXB_SWEEP=merge), which zero-copy graphs use.  CC / SSSP pull iterations run
    the flagged sweep (and the split, where it is on) with their own vertex programs, like PageRank.
The tolerance is wider than one wrong edge into a large hub; tests/test_gpu_exact.py compares the same paths bit for bit
on inputs where every summation order is exact."""
import numpy as np
import pytest

import oracle as O
import lux_b200 as L
from graphs import ALL_SMALL, rmat

pytestmark = pytest.mark.gpu
REL_TOL = 1e-6


def assert_close(gpu, ref):
    ref64 = ref.astype(np.float64)
    err = np.abs(gpu.astype(np.float64) - ref64)
    bad = np.nonzero(err > REL_TOL * np.abs(ref64))[0]
    assert bad.size == 0, "max rel err %.3e at %d (%d bad)" % ((err / np.maximum(np.abs(ref64), 1e-300)).max(), bad[0], bad.size)


def force(monkeypatch, bs, min_indeg, blocks=48, shape=0, main_shape=0):
    monkeypatch.setenv("LUXB_SB", "1")
    monkeypatch.setenv("LUXB_SB_BS", str(bs))
    monkeypatch.setenv("LUXB_SB_MIN_INDEG", str(min_indeg))
    monkeypatch.setenv("LUXB_SB_BLOCKS", str(blocks))
    monkeypatch.setenv("LUXB_SEG_PANEL_SHAPE", str(shape))
    monkeypatch.setenv("LUXB_SEG_MAIN_SHAPE", str(main_shape))


@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_panel_small_graphs(name, monkeypatch):
    force(monkeypatch, bs=16, min_indeg=2)
    row_end, src = ALL_SMALL[name]()
    for ni in (1, 3):
        assert_close(L.pagerank(row_end, src, num_iter=ni), O.pagerank(row_end, src, ni))


@pytest.mark.parametrize("bs,min_indeg,blocks,shape,main_shape", [(64, 4, 48, 0, 0), (256, 16, 8, 1, 1), (1024, 2, 64, 2, 2), (4096, 64, 3, 3, 3),
                                                                 (128, 1, 64, 4, 4), (32768, 8, 2, 5, 5)])
def test_panel_rmat16_parameter_sweep(bs, min_indeg, blocks, shape, main_shape, monkeypatch):
    force(monkeypatch, bs, min_indeg, blocks, shape, main_shape)
    row_end, src = rmat(16)
    with L.LuxGraph.from_csc(row_end, src) as g:
        g.init()
        st = g.stats()
        assert st["panel_edges"] > 0 and st["panel_hubs"] > 0 and 1 <= st["panel_blocks"] <= blocks
        g.iterate(10)
        assert_close(g.values(), O.pagerank(row_end, src, 10))


def test_panel_is_deterministic_and_off_switch_agrees(monkeypatch):
    row_end, src = rmat(15)
    force(monkeypatch, 128, 8)
    a = L.pagerank(row_end, src, num_iter=4)
    b = L.pagerank(row_end, src, num_iter=4)
    assert np.array_equal(a, b)
    monkeypatch.setenv("LUXB_SB", "0")
    with L.LuxGraph.from_csc(row_end, src) as g:
        g.init()
        assert g.stats()["panel_edges"] == 0
        g.iterate(4)
        c = g.values()
    assert_close(a, c.astype(np.float32))


def test_panel_default_parameters_rmat22_one_step():
    """Default (automatic) configuration on a partition large enough to switch the split on by itself."""
    scale = 22
    nv, ne = 1 << scale, 16 << scale
    with L.LuxGraph.from_rmat(scale, nv, ne, 27) as g:
        row_end, src = g.local_csc()
        g.init()
        st = g.stats()
        assert st["panel_edges"] > ne // 5, st
        g.iterate(2)
        x2 = g.values()
        deg = g.out_degree()
        g.iterate(1)
        x3 = g.values()
    assert_close(x3, O.pagerank_iter(row_end, src, deg, x2))


def test_panel_set_values_restart(monkeypatch):
    force(monkeypatch, 64, 4)
    row_end, src = rmat(14)
    with L.LuxGraph.from_csc(row_end, src) as g:
        g.init()
        g.iterate(2)
        x2 = g.values()
        g.iterate(3)
        x5 = g.values()
        g.set_values(x2)
        g.iterate(3)
        assert np.array_equal(g.values(), x5)


@pytest.mark.parametrize("main_shape", [0, 1, 2, 3, 4, 5, 6, 7])
def test_plain_seg_sweep_shapes(main_shape, monkeypatch):
    """The flagged stream without the split, every shape, on graphs with hubs spanning many pieces, empty vertices, no edges."""
    monkeypatch.setenv("LUXB_SB", "0")
    monkeypatch.setenv("LUXB_SEG_MAIN_SHAPE", str(main_shape))
    for name in ("star", "trailing_isolated", "no_edges", "rmat12_ragged_nv"):
        row_end, src = ALL_SMALL[name]()
        assert_close(L.pagerank(row_end, src, num_iter=3), O.pagerank(row_end, src, 3))
    row_end, src = rmat(17)
    assert_close(L.pagerank(row_end, src, num_iter=5), O.pagerank(row_end, src, 5))


def test_merge_path_sweep_still_available(monkeypatch):
    monkeypatch.setenv("LUXB_SWEEP", "merge")
    row_end, src = rmat(16)
    assert_close(L.pagerank(row_end, src, num_iter=5), O.pagerank(row_end, src, 5))


def test_local_values_roundtrip(monkeypatch):
    force(monkeypatch, 64, 4)
    row_end, src = rmat(14)
    with L.LuxGraph.from_csc(row_end, src) as g:
        g.init()
        g.iterate(2)
        x2 = g.local_values()
        assert np.array_equal(x2, g.values())  # one rank: the slice is everything
        g.iterate(3)
        x5 = g.values()
        g.set_local_values(x2)
        g.iterate(3)
        assert np.array_equal(g.local_values(), x5)
