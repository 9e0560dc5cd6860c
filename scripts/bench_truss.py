"""k-truss decomposition on the C4 graph (device-generated RMAT-24, edge factor 16, seed 24), on 1 GPU or on N GPUs
(re-launches itself under torch.distributed.run).  Prints ONE JSON line:

  card name and power limit (read in the same call); construction time (luxb_init, synchronised, support included);
  run time per luxb_truss_run (support count + peel; median and min over --reps runs after one warm-up run, luxb_stats
  loop_seconds); rounds, levels, kmax and the widest round; ms and kernel launches per round; with --oracle, parity
  against the CPU oracle (tests/truss_oracle.c: edges, support, τ and the round trace bit for bit) and its CPU time.

  With --profile, one more run under torch.profiler (CUDA activities, after the timed runs) gives the device time of
  every kernel of the run summed by name, the support kernels' sum ("support_ms") and the rest ("peel kernels").

  python scripts/bench_truss.py [--gpus N] [--scale 24] [--reps 5] [--oracle] [--profile]

Hardware bounds, at the data-sheet 3.35 TB/s: the support count makes one probe per (oriented edge (u, v), entry of
N+(v)), each a 4-byte read of an out-list entry (the same probes as triangle counting); the peel walks, for every edge
once, the shorter of its endpoints' lists, each entry an 8-byte (neighbour, edge id) read.  Both counts are computed on
the host from the edges; the binary searches and atomics come on top of either bound."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # the k-truss oracle lives with the tests
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_tc import DATASHEET_TBPS, card  # noqa: E402


def profile_run(g, torch):
    """Device time of every kernel of one more run, summed by kernel name, in ms."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.truss_run()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", None)
        if us is None:
            us = getattr(e, "self_cuda_time_total", 0.0)
        if not us:
            continue
        name = e.key
        for tag in ("truss_", "kcore_"):
            if tag in name:
                name = name[name.index(tag):].split("(")[0].split("<")[0]
                break
        else:
            if "cub" in name or "Scan" in name:
                name = "cub scan"
        out[name] = out.get(name, 0.0) + us / 1e3
    out["all kernels"] = sum(v for k, v in out.items())
    return {k: round(v, 3) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def work_counts(lo, hi, nv):
    """(support probes, peel walk entries): Σ |N+(v)| over the degree-oriented edges (u, v), and Σ min(deg u, deg v)."""
    deg = np.bincount(lo, minlength=nv) + np.bincount(hi, minlength=nv)
    a = deg[lo].astype(np.int64) << 32 | lo
    b = deg[hi].astype(np.int64) << 32 | hi
    head = np.where(a < b, hi, lo)  # the edge points from the lower (degree, id) to the higher one
    outdeg = np.bincount(np.where(a < b, lo, hi), minlength=nv)
    return int(outdeg[head].sum()), int(np.minimum(deg[lo], deg[hi]).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle", action="store_true")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.gpus > 1 and world == 1:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(args.gpus), "--master-addr",
               "127.0.0.1", "--master-port", os.environ.get("LUX_PORT", "29654")] + sys.argv
        return subprocess.call(cmd)
    rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    import torch
    import lux_b200 as L
    if world > 1:
        import torch.distributed as dist
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    scale, seed = args.scale, 24
    nv, ne = 1 << scale, 16 << scale
    name, power = card()
    result = dict(bench="truss", graph="RMAT-%d ef16 seed %d" % (scale, seed), nv=nv, ne=ne, gpus=world, card=name, power_limit=power)
    g = L.LuxGraph.from_rmat(scale, nv, ne, seed, app=L.APP_TRUSS, rank=rank, nranks=world, device=local)
    g.comm_init_torch()
    torch.cuda.synchronize(local)
    t0 = time.perf_counter()
    g.init()  # synchronises its stream before it returns
    result["construction_ms"] = 1e3 * (time.perf_counter() - t0)
    kmax = g.truss_run()  # warm-up
    times, launches = [], []
    for _ in range(max(args.reps, 1)):
        s0 = g.stats()
        assert g.truss_run() == kmax
        s1 = g.stats()
        times.append(s1["loop_seconds"] - s0["loop_seconds"])
        launches.append(s1["kernel_launches"] - s0["kernel_launches"])
    if world > 1:
        v = torch.tensor(times, dtype=torch.float64, device="cuda")
        dist.all_reduce(v, op=dist.ReduceOp.MAX)
        times = v.cpu().tolist()
    st = g.stats()
    runs = max(args.reps, 1) + 1
    rounds = st["iterations"] // runs
    active, pull = g.trace()
    lo, hi, sup, tau = g.truss_edges()
    kernels = profile_run(g, torch) if args.profile else None
    row_end, src = g.local_csc() if world == 1 else (None, None)
    g.close()
    med = float(np.median(times))
    probes, walk = work_counts(lo, hi, nv)
    support_bound = 4.0 * probes / (DATASHEET_TBPS * 1e12) * 1e3
    walk_bound = 8.0 * walk / (DATASHEET_TBPS * 1e12) * 1e3
    result.update(kmax=kmax, m=len(lo), triangles=int(sup.astype(np.int64).sum() // 3), rounds=rounds,
                  levels=int(len(np.unique(pull))), largest_round=int(active.max()) if len(active) else 0,
                  run_ms=dict(median=1e3 * med, min=1e3 * min(times), reps=len(times)), ms_per_round=1e3 * med / max(rounds, 1),
                  launches_per_round=float(np.median(launches)) / max(rounds, 1),
                  support_probes=probes, support_bound_ms_at_datasheet=support_bound,
                  peel_walk_entries=walk, peel_walk_bound_ms_at_datasheet=walk_bound)
    if kernels is not None:
        result["profiled_run_kernel_ms"] = kernels
        result["support_ms"] = round(sum(v for k, v in kernels.items() if k.startswith("truss_support")), 3)
        result["peel_kernels_ms"] = round(kernels["all kernels"] - result["support_ms"], 3)
    else:
        result["support_ms"] = "not measured (use --profile)"
    if rank == 0 and args.oracle:
        import oracle as O
        import truss_oracle as R
        if row_end is None:
            row_end, src = O.gen_rmat_csc(scale, nv, ne, seed)
        ref = R.run(row_end, src)
        result.update(oracle_cpu_s=ref["seconds"],
                      parity=bool(kmax == ref["kmax"] and rounds == ref["rounds"] and np.array_equal(lo, ref["lo"])
                                  and np.array_equal(hi, ref["hi"]) and np.array_equal(sup, ref["support"])
                                  and np.array_equal(tau, ref["truss"]) and np.array_equal(active, ref["trace_active"])
                                  and np.array_equal(pull, ref["trace_k"])))
    if rank == 0:
        print(json.dumps(result), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
