"""Worker for the multi-GPU triangle-counting test: run under torch.distributed.run, one rank per GPU.  Every rank opens
its partition of the same graph; luxb_init exchanges the distinct edge keys so that each rank holds the whole oriented
graph, each rank counts at the vertices of its range and t is summed over the ranks.  Every rank's t and T must equal
the one-rank result (and the oracle).  Cases: RMAT-16 from a CSC, RMAT-14 generated on the device, K_300 stored in both
directions, and a graph whose last partition holds vertices but no edges (asserted)."""
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
import tc_oracle as T  # noqa: E402
from mgpu_bc_worker import edge_free_case  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    cases = [("rmat16", *O.gen_rmat_csc(16, 1 << 16, 16 << 16, 27)), ("k300_both", *T.variant(*T.complete(300)[:2], "both")),
             ("edge_free_last_rank", *edge_free_case(world))]
    ok = True
    for name, row_end, src in cases + [("rmat14_device", None, None)]:
        if row_end is None:
            g = L.LuxGraph.from_rmat(14, 1 << 14, 16 << 14, 5, app=L.APP_TC, rank=rank, nranks=world, device=local)
        else:
            g = L.LuxGraph.from_csc(row_end, src, app=L.APP_TC, rank=rank, nranks=world, device=local, balanced=True)
        g.comm_init_torch()
        g.init()
        total = g.tc_run()
        t = g.values()
        local_t = g.local_values()
        b = g.bounds()
        edge_free = int(b["col_left"][-1]) == g.ne and int(b["row_right"][-1]) >= int(b["row_left"][-1])
        g.close()
        if row_end is None:
            with L.LuxGraph.from_rmat(14, 1 << 14, 16 << 14, 5, app=L.APP_PAGERANK, device=local) as h:
                row_end, src = h.local_csc()
        with L.LuxGraph.from_csc(row_end, src, app=L.APP_TC, device=local) as one:
            one.init()
            total1 = one.tc_run()
            t1 = one.values()
        ref = T.run(row_end, src)
        rl = int(b["row_left"][rank])
        good = total == total1 == ref["total"] and np.array_equal(t, t1) and np.array_equal(t, ref["t"])
        good = good and np.array_equal(local_t, t[rl:rl + len(local_t)])
        if name == "edge_free_last_rank":
            good = good and edge_free
        print("tc [%s] rank %d world=%d: T=%d %s%s" % (name, rank, world, total, "OK" if good else "FAIL",
                                                       " (last partition edge-free)" if edge_free else ""), flush=True)
        ok = ok and good
        dist.barrier()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("MGPU_TC %s" % ("PASS" if int(flag) else "FAIL"), flush=True)
    sys.exit(0 if int(flag) else 1)


if __name__ == "__main__":
    main()
