"""Worker for the multi-GPU k-truss test: run under torch.distributed.run, one rank per GPU.  Every rank opens its
partition of the same graph, counts the support at its own range (summed through NCCL), walks every round's F and lowers
its own edges; the pieces of F are exchanged through NCCL.  Every rank's edges, support, truss numbers, vertex truss,
kmax, trace and summed check() must equal the oracle's.  Cases: RMAT-14 from a CSC, RMAT-12 generated on the device,
disjoint cliques K_3 .. K_20, and a graph whose last partition holds vertices but no edges (asserted)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import lux_b200 as L  # noqa: E402
import oracle as O  # noqa: E402
import truss_oracle as R  # noqa: E402
from mgpu_bc_worker import edge_free_case  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    cases = [("rmat14", *O.gen_rmat_csc(14, 1 << 14, 16 << 14, 27)), ("cliques", *R.cliques(20)[:2]),
             ("edge_free_last_rank", *edge_free_case(world))]
    ok = True
    for name, row_end, src in cases + [("rmat12_device", None, None)]:
        if row_end is None:
            g = L.LuxGraph.from_rmat(12, 1 << 12, 16 << 12, 5, app=L.APP_TRUSS, rank=rank, nranks=world, device=local)
            row_end, src = None, None
        else:
            g = L.LuxGraph.from_csc(row_end, src, app=L.APP_TRUSS, rank=rank, nranks=world, device=local)
        g.comm_init_torch()
        g.init()
        kmax = g.truss_run()
        tv = g.values()
        edges = g.truss_edges()
        active, pull = g.trace()
        bad = torch.tensor([g.check()], device="cuda")
        dist.all_reduce(bad)
        b = g.bounds()
        edge_free = int(b["col_left"][-1]) == g.ne and int(b["row_right"][-1]) >= int(b["row_left"][-1])
        g.close()
        if row_end is None:
            with L.LuxGraph.from_rmat(12, 1 << 12, 16 << 12, 5, app=L.APP_PAGERANK, device=local) as h:
                row_end, src = h.local_csc()
        ref = R.run(row_end, src)
        good = kmax == ref["kmax"] and np.array_equal(tv, ref["vertex"]) and int(bad) == 0
        good = good and all(np.array_equal(x, ref[k]) for x, k in zip(edges, ("lo", "hi", "support", "truss")))
        good = good and np.array_equal(active, ref["trace_active"]) and np.array_equal(pull, ref["trace_k"])
        if name == "edge_free_last_rank":
            good = good and edge_free
        print("truss [%s] rank %d world=%d: kmax=%d rounds=%d %s%s" % (name, rank, world, kmax, len(active),
                                                                           "OK" if good else "FAIL",
                                                                           " (last partition edge-free)" if edge_free else ""), flush=True)
        ok = ok and good
        dist.barrier()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("MGPU_TRUSS %s" % ("PASS" if int(flag) else "FAIL"), flush=True)
    sys.exit(0 if int(flag) else 1)


if __name__ == "__main__":
    main()
