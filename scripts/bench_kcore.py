"""k-core decomposition on the C4 graph (device-generated RMAT-24, edge factor 16, seed 24), on 1 GPU or on N GPUs
(re-launches itself under torch.distributed.run).  Prints ONE JSON line:

  card name and power limit (read in the same call); construction time (luxb_init, synchronised); run time per
  luxb_kcore_run (median and min over --reps runs after one warm-up run, luxb_stats loop_seconds); rounds, levels and
  the degeneracy; ms and kernel launches per round; and from the CPU oracle (tests/kcore_oracle.c) its CPU time and a
  parity flag (core, degeneracy and the round trace bit for bit).

  With --profile, one more run under torch.profiler (CUDA activities, after the timed runs) gives the device time of
  every kernel of the run summed by name, and the sum of all of them (the rest of the run is gaps: launches and the
  host synchronisation of every round).

  python scripts/bench_kcore.py [--gpus N] [--scale 24] [--reps 5] [--no-oracle] [--profile]

Hardware bounds, at the data-sheet 3.35 TB/s: the peel reads every adjacency entry once, 2m x 4 bytes; the tally after
every round reads the alive list as it stood, with core and deg of each entry (12 bytes), and writes the survivors (4
bytes), summed over the rounds from the trace.  Each round also costs a host synchronisation and a few launches, which
neither bound includes; per-round time against them says which dominates."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # the k-core oracle lives with the tests
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_tc import DATASHEET_TBPS, card  # noqa: E402


def profile_run(g, torch):
    """Device time of every kernel of one more run, summed by kernel name (kcore kernels by their short name), in ms."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.kcore_run()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", None)
        if us is None:
            us = getattr(e, "self_cuda_time_total", 0.0)
        if not us:
            continue
        name = e.key
        if "kcore_" in name:
            name = name[name.index("kcore_"):].split("(")[0].split("<")[0]
        elif "cub" in name or "Scan" in name:
            name = "cub scan"
        out[name] = out.get(name, 0.0) + us / 1e3
    out["all kernels"] = sum(v for k, v in out.items())
    return {k: round(v, 3) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.gpus > 1 and world == 1:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(args.gpus), "--master-addr",
               "127.0.0.1", "--master-port", os.environ.get("LUX_PORT", "29653")] + sys.argv
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
    result = dict(bench="kcore", graph="RMAT-%d ef16 seed %d" % (scale, seed), nv=nv, ne=ne, gpus=world, card=name, power_limit=power)
    g = L.LuxGraph.from_rmat(scale, nv, ne, seed, app=L.APP_KCORE, rank=rank, nranks=world, device=local)
    g.comm_init_torch()
    torch.cuda.synchronize(local)
    t0 = time.perf_counter()
    g.init()  # synchronises its stream before it returns
    result["construction_ms"] = 1e3 * (time.perf_counter() - t0)
    degeneracy = g.kcore_run()  # warm-up
    times, launches = [], []
    for _ in range(max(args.reps, 1)):
        s0 = g.stats()
        assert g.kcore_run() == degeneracy
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
    two_m = st["edges_processed"] // runs
    active, pull = g.trace()
    core = g.values()
    kernels = profile_run(g, torch) if args.profile else None
    row_end, src = g.local_csc() if world == 1 else (None, None)
    g.close()
    med = float(np.median(times))
    bound_ms = 4.0 * two_m / (DATASHEET_TBPS * 1e12) * 1e3
    # alive vertices (over all ranks) before each round and after it; the first tally is over every vertex
    after = nv - np.cumsum(active.astype(np.int64))
    before = np.concatenate([[nv], after[:-1]])
    tally_bytes = 16 * nv + int((12 * before + 4 * after).sum())
    tally_ms = tally_bytes / (DATASHEET_TBPS * 1e12) * 1e3
    result.update(degeneracy=degeneracy, rounds=rounds, levels=int(len(np.unique(pull))), largest_round=int(active.max()),
                  adjacency_entries=two_m, run_ms=dict(median=1e3 * med, min=1e3 * min(times), reps=len(times)),
                  ms_per_round=1e3 * med / rounds, launches_per_round=float(np.median(launches)) / rounds,
                  adjacency_pass_bound_ms_at_datasheet=bound_ms, adjacency_pass_fraction_of_datasheet=bound_ms / (1e3 * med),
                  tally_bytes=tally_bytes, tally_bound_ms_at_datasheet=tally_ms,
                  both_bounds_fraction_of_datasheet=(bound_ms + tally_ms) / (1e3 * med))
    if kernels is not None:
        result["profiled_run_kernel_ms"] = kernels
    if rank == 0 and not args.no_oracle:
        import oracle as O
        import kcore_oracle as K
        if row_end is None:
            row_end, src = O.gen_rmat_csc(scale, nv, ne, seed)
        ref = K.run(row_end, src)
        result.update(oracle_cpu_s=ref["seconds"],
                      parity=bool(degeneracy == ref["degeneracy"] and rounds == ref["rounds"] and two_m == 2 * ref["m"]
                                  and np.array_equal(core, ref["core"]) and np.array_equal(active, ref["trace_active"])
                                  and np.array_equal(pull, ref["trace_k"])))
    if rank == 0:
        print(json.dumps(result), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
