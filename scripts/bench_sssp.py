"""Weighted vs unweighted SSSP on the same graph: RMAT-`scale` (edge factor 16, seed 24, -start 0; C4 at scale 24),
device-generated, on 1 GPU or on N GPUs (re-launches itself under torch.distributed.run).  Prints ONE JSON line:

  card name and power limit (read in the same call), and per mode (unweighted = hop counts, weighted = weights 1..255):
  iterations, pull iterations, loop seconds (luxb_stats, median / min over --reps runs), edges scanned (Σ over ranks),
  MTEPS as ne / t and as Σ scanned / t (SURVEY §8d), and a parity flag against the CPU oracle run with P = ranks
  (labels, iteration count and per-iteration trace), with the oracle's CPU time and core count.

  python scripts/bench_sssp.py [--gpus N] [--scale 24] [--reps 3] [--no-oracle]

Push-step bytes are 20·active + 12·edges_scanned + frontier for weighted SSSP (8 B per edge for the unweighted one:
the weight adds 4 B per scanned edge)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # the weighted-SSSP oracle lives with the tests


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return name, power
    except Exception:  # noqa: BLE001
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-oracle", action="store_true")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.gpus > 1 and world == 1:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(args.gpus), "--master-addr",
               "127.0.0.1", "--master-port", os.environ.get("LUX_PORT", "29631")] + sys.argv
        return subprocess.call(cmd)
    rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    import torch
    import lux_b200 as L
    if world > 1:
        import torch.distributed as dist
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    scale, seed, start = args.scale, 24, 0
    nv, ne = 1 << scale, 16 << scale
    name, power = card()
    result = dict(bench="sssp_weighted_vs_unweighted", graph="RMAT-%d ef16 seed %d start %d" % (scale, seed, start), nv=nv, ne=ne,
                  gpus=world, card=name, power_limit=power)
    labels = {}
    for mode, app in (("unweighted", L.APP_SSSP), ("weighted", L.APP_SSSP_WEIGHTED)):
        times, scanned = [], []
        for _ in range(max(args.reps, 1)):
            g = L.LuxGraph.from_rmat(scale, nv, ne, seed, app=app, rank=rank, nranks=world, device=local, start=start,
                                     exchange=L.EXCHANGE_P2P if world > 1 else L.EXCHANGE_NCCL)
            g.comm_init_torch()
            g.init()
            if world > 1:
                g.p2p_connect_torch()
            it = g.run_to_convergence()
            st = g.stats()
            t = st["loop_seconds"]
            sc = st["edges_processed"]
            if world > 1:
                v = torch.tensor([t, float(sc)], dtype=torch.float64, device="cuda")
                tmax = v[:1].clone()
                dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
                dist.all_reduce(v[1:], op=dist.ReduceOp.SUM)
                t, sc = float(tmax), int(v[1])
            times.append(t)
            scanned.append(sc)
            lab = g.values()
            trace = g.trace()
            g.close()
            if world > 1:
                dist.barrier()
        t_med = float(np.median(times))
        labels[mode] = (lab, it, trace)
        result[mode] = dict(iterations=it, pull_iterations=int(st["pull_iterations"]), loop_s_median=t_med, loop_s_min=min(times),
                            ms_to_convergence=1e3 * t_med, edges_scanned=int(scanned[0]),
                            mteps_ne=ne / t_med / 1e6, mteps_scanned=scanned[0] / t_med / 1e6, reps=len(times))
    if rank == 0 and not args.no_oracle:
        import oracle as O
        import weighted_oracle as W
        t0 = time.perf_counter()
        row_end, src = O.gen_rmat_csc(scale, nv, ne, seed)
        w = W.rmat_weights(seed, row_end, src)
        t_gen = time.perf_counter() - t0
        for mode in ("unweighted", "weighted"):
            t0 = time.perf_counter()
            if mode == "weighted":
                ref = W.label_run(row_end, src, w, P=world, start=start)
            else:
                ref = O.label_run(O.APP_SSSP, row_end, src, P=world, start=start)
            t_or = time.perf_counter() - t0
            lab, it, (active, pull) = labels[mode]
            result[mode]["parity"] = bool(np.array_equal(lab, ref["labels"]) and it == ref["iters"] and
                                          np.array_equal(active, ref["active"]) and np.array_equal(pull, ref["pull"]))
            result[mode]["oracle_cpu_s"] = t_or
        result["oracle_gen_s"] = t_gen
        result["oracle_threads"] = O.num_threads()
        result["host_cpus"] = os.cpu_count()
    if rank == 0:
        print(json.dumps(result), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
