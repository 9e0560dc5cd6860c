"""Worker for the multi-GPU weighted-SSSP parity test: run under torch.distributed.run, one rank per GPU.  Every rank
opens its partition of the same weighted RMAT graph (device generator, and host CSC arrays), exchanges frontiers by
NCCL and by P2P pushes, and the result must equal the oracle run with P = world partitions."""
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
import weighted_oracle as W  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    scale, seed = 16, 27
    nv, ne = 1 << scale, 16 << scale
    row_end, src = O.gen_rmat_csc(scale, nv, ne, seed)
    w = W.rmat_weights(seed, row_end, src)
    ref = W.label_run(row_end, src, w, P=world, start=0)
    ok = True
    for opener, oname in ((lambda ex: L.LuxGraph.from_rmat(scale, nv, ne, seed, app=L.APP_SSSP_WEIGHTED, rank=rank, nranks=world,
                                                             device=local, start=0, exchange=ex), "rmat"),
                          (lambda ex: L.LuxGraph.from_csc(row_end, src, w, app=L.APP_SSSP_WEIGHTED, rank=rank, nranks=world,
                                                            device=local, start=0, exchange=ex), "csc")):
        for exchange, ename in ((L.EXCHANGE_NCCL, "nccl"), (L.EXCHANGE_P2P, "p2p push")):
            g = opener(exchange)
            g.comm_init_torch()
            g.init()
            connected = exchange == L.EXCHANGE_NCCL or g.p2p_connect_torch()
            it = g.run_to_convergence()
            lab = g.values()
            bad = torch.tensor([g.check()], dtype=torch.int64, device="cuda")
            dist.all_reduce(bad)
            active, pull = g.trace()
            good = (connected and np.array_equal(lab, ref["labels"]) and int(bad) == 0 and it == ref["iters"]
                    and np.array_equal(active, ref["active"]) and np.array_equal(pull, ref["pull"]))
            if rank == 0:
                print("weighted sssp [%s, %s] world=%d: %s (iters %d vs %d)" % (oname, ename, world, "OK" if good else "FAIL", it,
                                                                                 ref["iters"]), flush=True)
            ok = ok and good
            g.close()
            dist.barrier()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("MGPU_SSSP_W %s" % ("PASS" if int(flag) else "FAIL"), flush=True)
    sys.exit(0 if int(flag) else 1)


if __name__ == "__main__":
    main()
