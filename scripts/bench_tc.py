"""Triangle counting on the C4 graph (device-generated RMAT-24, edge factor 16, seed 24), on 1 GPU or on N GPUs
(re-launches itself under torch.distributed.run).  Prints ONE JSON line:

  card name and power limit (read in the same call); construction time (luxb_init, synchronised); count time per
  luxb_tc_run (median and min over --reps runs after one warm-up run, luxb_stats loop_seconds); T and m; and from the
  CPU oracle (tests/tc_oracle.c) the largest out-degree, the probe count sum over oriented (u, v) of |N+(v)|, its CPU
  time and thread count, and a parity flag (t and T bit for bit); probes per second of the device count.

  python scripts/bench_tc.py [--gpus N] [--scale 24] [--reps 5] [--no-oracle]

Hardware bound: one pass over the oriented CSR, 4 m + 8 n bytes, at the data-sheet 3.35 TB/s.  The count re-reads the
out-lists once per probe and mostly hits L2, so this bound is loose; it is stated as a fraction of the data sheet."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # the TC oracle lives with the tests
DATASHEET_TBPS = 3.35  # H100 SXM5 80 GB HBM3


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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.gpus > 1 and world == 1:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(args.gpus), "--master-addr",
               "127.0.0.1", "--master-port", os.environ.get("LUX_PORT", "29643")] + sys.argv
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
    result = dict(bench="tc", graph="RMAT-%d ef16 seed %d" % (scale, seed), nv=nv, ne=ne, gpus=world, card=name, power_limit=power)
    g = L.LuxGraph.from_rmat(scale, nv, ne, seed, app=L.APP_TC, rank=rank, nranks=world, device=local)
    g.comm_init_torch()
    torch.cuda.synchronize(local)
    t0 = time.perf_counter()
    g.init()  # synchronises its stream before it returns
    result["construction_ms"] = 1e3 * (time.perf_counter() - t0)
    total = g.tc_run()  # warm-up
    times = []
    for _ in range(max(args.reps, 1)):
        s0 = g.stats()["loop_seconds"]
        assert g.tc_run() == total
        times.append(g.stats()["loop_seconds"] - s0)
    if world > 1:
        v = torch.tensor(times, dtype=torch.float64, device="cuda")
        dist.all_reduce(v, op=dist.ReduceOp.MAX)
        times = v.cpu().tolist()
    st = g.stats()
    m = st["edges_processed"] // st["iterations"]
    t = g.values()
    row_end, src = g.local_csc() if world == 1 else (None, None)
    g.close()
    med = float(np.median(times))
    bound_ms = (4.0 * m + 8.0 * nv) / (DATASHEET_TBPS * 1e12) * 1e3
    result.update(triangles=total, m=m, count_ms=dict(median=1e3 * med, min=1e3 * min(times), reps=len(times)),
                  csr_pass_bound_ms_at_datasheet=bound_ms, csr_pass_fraction_of_datasheet=bound_ms / (1e3 * med))
    if rank == 0 and not args.no_oracle:
        import oracle as O
        import tc_oracle as T
        if row_end is None:
            row_end, src = O.gen_rmat_csc(scale, nv, ne, seed)
        ref = T.run(row_end, src)
        result.update(max_out_degree=ref["max_out"], probes=ref["probes"], probes_per_s=ref["probes"] / med,
                      oracle_cpu_s=ref["seconds"], oracle_threads=ref["threads"], host_cpus=os.cpu_count(),
                      parity=bool(total == ref["total"] and m == ref["m"] and np.array_equal(t, ref["t"])))
    if rank == 0:
        print(json.dumps(result), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
