"""Worker for the multi-GPU k-core test: run under torch.distributed.run, one rank per GPU.  Every rank opens its
partition of the same graph, peels its own range and exchanges each round's pieces through NCCL.  Every rank's core
numbers, degeneracy, trace and summed check() must equal the oracle's.  Cases: RMAT-16 from a CSC, RMAT-14 generated on
the device, a chain of cliques K_2 .. K_60, and a graph whose last partition holds vertices but no edges (asserted)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import kcore_oracle as K  # noqa: E402
import lux_b200 as L  # noqa: E402
import oracle as O  # noqa: E402
from mgpu_bc_worker import edge_free_case  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    cases = [("rmat16", *O.gen_rmat_csc(16, 1 << 16, 16 << 16, 27)), ("clique_chain", *K.clique_chain(2, 60)[:2]),
             ("edge_free_last_rank", *edge_free_case(world))]
    ok = True
    for name, row_end, src in cases + [("rmat14_device", None, None)]:
        if row_end is None:
            g = L.LuxGraph.from_rmat(14, 1 << 14, 16 << 14, 5, app=L.APP_KCORE, rank=rank, nranks=world, device=local)
            row_end, src = None, None
        else:
            g = L.LuxGraph.from_csc(row_end, src, app=L.APP_KCORE, rank=rank, nranks=world, device=local)
        g.comm_init_torch()
        g.init()
        degeneracy = g.kcore_run()
        core = g.values()
        active, pull = g.trace()
        bad = torch.tensor([g.check()], device="cuda")
        dist.all_reduce(bad)
        b = g.bounds()
        edge_free = int(b["col_left"][-1]) == g.ne and int(b["row_right"][-1]) >= int(b["row_left"][-1])
        g.close()
        if row_end is None:
            with L.LuxGraph.from_rmat(14, 1 << 14, 16 << 14, 5, app=L.APP_PAGERANK, device=local) as h:
                row_end, src = h.local_csc()
        ref = K.run(row_end, src)
        good = degeneracy == ref["degeneracy"] and np.array_equal(core, ref["core"]) and int(bad) == 0
        good = good and np.array_equal(active, ref["trace_active"]) and np.array_equal(pull, ref["trace_k"])
        if name == "edge_free_last_rank":
            good = good and edge_free
        print("kcore [%s] rank %d world=%d: degeneracy=%d rounds=%d %s%s" % (name, rank, world, degeneracy, len(active),
                                                                           "OK" if good else "FAIL",
                                                                           " (last partition edge-free)" if edge_free else ""), flush=True)
        ok = ok and good
        dist.barrier()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("MGPU_KCORE %s" % ("PASS" if int(flag) else "FAIL"), flush=True)
    sys.exit(0 if int(flag) else 1)


if __name__ == "__main__":
    main()
