"""Executable models (numpy, CPU) of the pull sweeps' cross-tile fix-up in lux_b200/csrc/pull.cuh, checked against the
obvious sequential definition: carry into tile t = sum of the tail partials of the tiles since, and including, the last
tile before t that completed a vertex.
  * the three-kernel segmented scan (pull_fixup_scan / _blocks / _apply, LUXB_FUSED_FIXUP=0): 256-tile blocks, 1024
    serial chunks + shuffle scans, including n_blocks > 1024 (chunk length > 1);
  * the fused chained scan (pull_fixup_fused_kernel, the default): in-block shuffle scan, then a decoupled look-back
    over the predecessors' published aggregates / inclusive prefixes, with the publication state each predecessor may
    be in when a block looks back (prefix published, or only the aggregate) and status words left by earlier launches.
They mirror the CUDA control flow so that a change of the kernels' structure has a CPU-side regression check of the
algebra.  Tails are integers: every summation order is exact, so the models must equal the definition bit for bit."""
import numpy as np
import pytest

FIX_BLOCK = 256


def comb(f2, v2, f1, v1):
    """(f1, v1) earlier, (f2, v2) later — seg_combine in pull.cuh."""
    return (f2 | f1, v2 if f2 else v1 + v2)


def seq_scan_exclusive(flags, vals):
    out_f, out_v = [], []
    f, v = 0, 0.0
    for ff, vv in zip(flags, vals):
        out_f.append(f)
        out_v.append(v)
        f, v = comb(int(ff), float(vv), f, v)
    return out_f, out_v, (f, v)


def model_fixup(flags, tails):
    n = len(flags)
    nb = (n + FIX_BLOCK - 1) // FIX_BLOCK
    carry_f, carry_v, agg = [0] * n, [0.0] * n, []
    for b in range(nb):  # pull_fixup_scan_kernel: exclusive in-block scan + block aggregate
        lo, hi = b * FIX_BLOCK, min(n, (b + 1) * FIX_BLOCK)
        ef, ev, total = seq_scan_exclusive(flags[lo:hi], tails[lo:hi])
        carry_f[lo:hi], carry_v[lo:hi] = ef, ev
        agg.append(total)
    # pull_fixup_blocks_kernel: 1024 threads, serial chunk of `per` blocks each, scan of chunk aggregates, rewrite
    per = (nb + 1023) // 1024
    chunk = []
    for k in range(1024):
        b0, b1 = min(k * per, nb), min(min(k * per, nb) + per, nb)
        f, v = 0, 0.0
        for b in range(b0, b1):
            f, v = comb(agg[b][0], agg[b][1], f, v)
        chunk.append((f, v))
    # two-level inclusive scan over the 1024 chunk aggregates (warps of 32, then warp aggregates)
    incl = []
    for w in range(32):
        f, v = 0, 0.0
        for lane in range(32):
            f, v = comb(chunk[w * 32 + lane][0], chunk[w * 32 + lane][1], f, v)
            incl.append((f, v))
    prefix = []
    for k in range(1024):
        w, lane = divmod(k, 32)
        wf, wv = 0, 0.0
        for ww in range(w):
            wf, wv = comb(incl[ww * 32 + 31][0], incl[ww * 32 + 31][1], wf, wv)
        pf, pv = (0, 0.0) if lane == 0 else incl[k - 1]
        prefix.append(comb(pf, pv, wf, wv))
    block_prefix = [None] * nb
    for k in range(1024):
        b0, b1 = min(k * per, nb), min(min(k * per, nb) + per, nb)
        pf, pv = prefix[k]
        for b in range(b0, b1):
            block_prefix[b] = (pf, pv)
            pf, pv = comb(agg[b][0], agg[b][1], pf, pv)
    # pull_fixup_apply_kernel
    out = []
    for t in range(n):
        c = carry_v[t] if carry_f[t] else block_prefix[t // FIX_BLOCK][1] + carry_v[t]
        out.append(c)
    return np.array(out)


@pytest.mark.parametrize("n,density", [(1, 1.0), (255, 0.5), (256, 0.0), (257, 0.01), (5000, 0.02), (300000, 0.0005), (300000, 0.3)])
def test_fixup_model_equals_sequential_definition(n, density):
    rng = np.random.default_rng(n)
    flags = (rng.random(n) < density).astype(np.int64)
    tails = rng.integers(0, 100, n).astype(np.float64)  # integers: every summation order is exact
    want = np.array(seq_scan_exclusive(flags, tails)[1])
    got = model_fixup(flags, tails)
    assert np.array_equal(got, want)


def warp_scan_inclusive(f, v):
    """Segmented inclusive scan over the last axis (32 lanes) with shfl_up steps, as the fix-up kernels run it."""
    lane = np.arange(32)
    for off in (1, 2, 4, 8, 16):
        pf = np.zeros_like(f)
        pv = np.zeros_like(v)
        pf[..., off:], pv[..., off:] = f[..., :-off], v[..., :-off]
        take = lane >= off  # seg_combine(sf, sv, pf, pv) on lanes >= off
        v = np.where(take & (f == 0), pv + v, v)
        f = np.where(take, f | pf, f)
    return f, v


def model_fused_fixup(flags, tails, rng, p_prefix, epoch=7, stop_after_one=False):
    """pull_fixup_fused_kernel: returns the carry into every tile.  Blocks run in ticket order; when block b looks back,
    each predecessor has published its aggregate and, with probability p_prefix, already its inclusive prefix.  A
    prefix slot not yet written in this launch holds the status word and value an earlier launch left there.
    stop_after_one: a deliberately wrong look-back that reads one predecessor only (the model's own sensitivity check)."""
    n = len(flags)
    nb = (n + FIX_BLOCK - 1) // FIX_BLOCK
    F = np.zeros(nb * FIX_BLOCK, np.int64)
    V = np.zeros(nb * FIX_BLOCK, np.float64)
    F[:n], V[:n] = flags, tails
    sf, sv = warp_scan_inclusive(F.reshape(nb, 8, 32), V.reshape(nb, 8, 32))
    wf, wv = np.zeros((nb, 8), np.int64), np.zeros((nb, 8), np.float64)  # aggregate of the preceding warps
    for w in range(1, 8):
        a_f, a_v = sf[:, w - 1, 31], sv[:, w - 1, 31]
        wv[:, w] = np.where(a_f == 0, wv[:, w - 1] + a_v, a_v)
        wf[:, w] = a_f | wf[:, w - 1]
    ef, ev = np.zeros_like(sf), np.zeros_like(sv)  # exclusive in-block prefix of each tile
    ef[..., 1:], ev[..., 1:] = sf[..., :-1], sv[..., :-1]
    ev = np.where(ef == 0, wv[..., None] + ev, ev)
    ef = ef | wf[..., None]
    af = sf[:, 7, 31] | wf[:, 7]  # block aggregates
    av = np.where(sf[:, 7, 31] == 0, wv[:, 7] + sv[:, 7, 31], sv[:, 7, 31])
    # chain slots: 2b = aggregate, 2b + 1 = inclusive prefix; status = (epoch << 2) | (flag << 1) | 1
    value = rng.integers(-1000, 1000, 2 * nb).astype(np.float64)  # left by an earlier launch
    status = ((epoch - 1) << 2) | (rng.integers(0, 2, 2 * nb) << 1) | 1
    prefix_f, prefix_v, prefix_visible = np.zeros(nb, np.int64), np.zeros(nb), np.zeros(nb, bool)
    bp_f, bp_v = np.zeros(nb, np.int64), np.zeros(nb)
    for b in range(nb):
        value[2 * b] = av[b]
        status[2 * b] = (epoch << 2) | (int(af[b]) << 1) | 1
        # what the predecessors have published by now: the real prefix, or still the stale slot of an earlier launch
        for q in range(b):
            if not prefix_visible[q] and rng.random() < p_prefix:
                prefix_visible[q] = True
                value[2 * q + 1] = prefix_v[q]
                status[2 * q + 1] = (epoch << 2) | (int(prefix_f[q]) << 1) | 1
        pf, pv = 0, 0.0
        q = b - 1
        while q >= 0 and not pf:
            have_prefix = (status[2 * q + 1] >> 2) == epoch
            s = status[2 * q + 1] if have_prefix else status[2 * q]
            qf, qv = int((s >> 1) & 1), value[2 * q + (1 if have_prefix else 0)]
            pv = pv if pf else qv + pv
            pf |= qf
            if have_prefix or stop_after_one:
                break
            q -= 1
        bp_f[b], bp_v[b] = pf, pv
        prefix_f[b] = int(af[b]) | pf
        prefix_v[b] = av[b] if af[b] else pv + av[b]
    carry = np.where(ef == 0, bp_v[:, None, None] + ev, ev)
    return carry.reshape(-1)[:n]


@pytest.mark.parametrize("n,density,p_prefix", [(1, 1.0, 0.5), (257, 0.01, 0.0), (5000, 0.0, 0.3), (5000, 0.02, 1.0),
                                                (40000, 0.001, 0.5), (40000, 0.0005, 0.0), (60000, 0.3, 0.2)])
def test_fused_fixup_model_equals_sequential_definition(n, density, p_prefix):
    rng = np.random.default_rng(n + int(100 * p_prefix))
    flags = (rng.random(n) < density).astype(np.int64)
    tails = rng.integers(0, 100, n).astype(np.float64)
    want = np.array(seq_scan_exclusive(flags, tails)[1])
    got = model_fused_fixup(flags, tails, rng, p_prefix)
    assert np.array_equal(got, want)


def test_fused_fixup_model_sees_a_broken_look_back():
    """The check is not vacuous: a look-back that stops after one predecessor's aggregate without a completed vertex
    (instead of walking on to a published prefix or a flagged aggregate) drops the carry that crosses several blocks."""
    n = 4 * FIX_BLOCK
    flags = np.zeros(n, np.int64)
    flags[10] = 1
    tails = np.ones(n)
    want = np.array(seq_scan_exclusive(flags, tails)[1])
    assert np.array_equal(model_fused_fixup(flags, tails, np.random.default_rng(0), 0.0), want)
    got = model_fused_fixup(flags, tails, np.random.default_rng(0), 0.0, stop_after_one=True)
    assert not np.array_equal(got, want)
    assert np.array_equal(got[:2 * FIX_BLOCK], want[:2 * FIX_BLOCK])
