"""GPU: betweenness centrality (LUXB_BC, LUXB_BC_WEIGHTED) on inputs whose path counts outgrow fp32 (wide_bc_inputs),
against the CPU oracles (tests/bc_oracle.c, tests/bc_weighted_oracle.c).

The suite's other BC inputs keep every sigma below 2^24 or make it a power of two, where fp32 holds every term and
partial of the sigma sums; these do not (tests/test_bc_wide_model.py shows on the CPU that a model of the device with any
one sigma step narrowed to fp32 fails them, and passes the older inputs).
  * the layered DAG (sigma up to 2^45, integers below 2^53; in-degree hubs of SEG, SEG + 1, 2 SEG + 1, 3 SEG + 1 and
    30 000 edges at sigma 2^35 to 2^38, an out-degree hub past SEG): lev / D and sigma bit for bit, delta and the scores
    at rtol 1e-10 with exact zeros;
  * the 500 x 500 directed lattice (sigma up to 2^992.7; every sum has at most two non-zero terms; hubs of SEG, SEG + 1
    and 3 SEG + 1 in- and out-edges with the lattice edges in chosen segments): lev / D, sigma, delta and the scores
    bit for bit.
Each from the root / corner, from an interior vertex, then a list of three sources in one bc_run (the scores add up over
every source run on the handle, in order); in the default configuration, with LUXB_SWEEP=merge and with zero-copy
edges; and at 2, 3 and 4 emulated ranks (the level pieces, the sigma broadcasts and the delta all-reduce straddle the
ranks)."""
import functools

import numpy as np
import pytest

import lux_b200 as L
import bc_oracle as B
import bc_weighted_oracle as BW
from emu_ranks import emulate, run_ranks
from wide_bc_inputs import lattice, layered, wide_count

pytestmark = pytest.mark.gpu
CASES = [(name, weighted) for name in ("layered", "lattice") for weighted in (False, True)]


@functools.lru_cache(maxsize=None)
def case(name, weighted):
    """The input and the oracle's answers: the states of the root and the interior source, then the state of the last
    source and the scores after the root, the interior source and the three-source list in that order."""
    f = layered(weighted) if name == "layered" else lattice(weighted)
    args = (f["row_end"], f["src"]) + ((f["weight"],) if weighted else ())
    run = (lambda srcs: BW.run(*args, srcs)) if weighted else (lambda srcs: B.run(*args, srcs))
    S = f["sources"]
    refs = {k: run([S[k]]) for k in ("root", "interior")}
    refs["multi"] = run(np.concatenate([[S["root"], S["interior"]], S["multi"]]).astype(np.uint32))
    return f, refs


def first_diff(got, want, what):
    """Bit for bit (floats by their bits), naming the first differing index."""
    g, w = np.asarray(got), np.asarray(want)
    if g.dtype.kind == "f":
        g, w = g.view(np.uint64), w.astype(np.float64).view(np.uint64)
    bad = np.nonzero(g != w)[0]
    assert bad.size == 0, "%s: %d values differ, first at %d: got %r, want %r" % (what, bad.size, bad[0], got[bad[0]], want[bad[0]])


def close(got, want, what):
    bad = np.nonzero(~np.isclose(got, want, rtol=1e-10, atol=0) | ((got == 0) != (want == 0)))[0]
    assert bad.size == 0, "%s: %d values off by more than rtol 1e-10, first at %d: got %r, want %r" % (
        what, bad.size, bad[0], got[bad[0]], want[bad[0]])


def check(name, weighted, state, ref, what, scores=None):
    lev, sigma, delta = state
    first_diff(lev, ref["dist"] if weighted else ref["lev"], what + " lev")
    first_diff(sigma, ref["sigma"], what + " sigma")
    if name == "lattice":  # every sum has at most two non-zero terms: one rounding whatever the order
        first_diff(delta, ref["delta"], what + " delta")
        if scores is not None:
            first_diff(scores, ref["scores"], what + " scores")
    else:                  # exact integer sigma; delta sums many quotients in the device's order
        assert ref["sigma"].max() < 2.0 ** 53, what
        close(delta, ref["delta"], what + " delta")
        if scores is not None:
            close(scores, ref["scores"], what + " scores")


def run_sources(g, f, refs, name, weighted, what):
    S = f["sources"]
    for k in ("root", "interior"):
        g.bc_run([S[k]])
        check(name, weighted, g.bc_source_state(), refs[k], "%s %s" % (what, k))
    g.bc_run(S["multi"])
    check(name, weighted, g.bc_source_state(), refs["multi"], what + " multi", g.values())


@pytest.mark.parametrize("name,weighted", CASES)
@pytest.mark.parametrize("config", ["default", "merge", "zero_copy"])
def test_wide_sigma(name, weighted, config, monkeypatch):
    if config == "merge":
        monkeypatch.setenv("LUXB_SWEEP", "merge")
    f, refs = case(name, weighted)
    assert wide_count(refs["root"]["sigma"]) > (5000 if name == "layered" else 240000)
    what = "%s%s %s" % ("weighted " if weighted else "", name, config)
    with L.LuxGraph.from_csc(f["row_end"], f["src"], f["weight"], app=L.APP_BC_WEIGHTED if weighted else L.APP_BC,
                             zero_copy=config == "zero_copy") as g:
        g.init()
        run_sources(g, f, refs, name, weighted, what)


def case_ranks(world, name, weighted):
    """Every rank runs the three source sets on its partition; each rank's full state and scores against the oracle."""
    f, refs = case(name, weighted)
    what = "%s%s" % ("weighted " if weighted else "", name)

    def body(rank, uid):
        g = L.LuxGraph.from_csc(f["row_end"], f["src"], f["weight"], app=L.APP_BC_WEIGHTED if weighted else L.APP_BC, rank=rank,
                                nranks=world, device=0)
        with g:
            g.comm_init(uid(0))
            g.init()
            run_sources(g, f, refs, name, weighted, "%s rank %d/%d" % (what, rank, world))

    run_ranks(world, body)


@pytest.mark.parametrize("name,weighted", CASES)
def test_wide_sigma_emulated_ranks(name, weighted):
    rc, out = emulate("test_gpu_bc_wide", "case_ranks", worlds=[2, 3, 4], name=name, weighted=weighted)
    assert rc == 0, out[-6000:]
