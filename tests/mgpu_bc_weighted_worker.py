"""Worker for the multi-GPU weighted betweenness-centrality test: run under torch.distributed.run, one rank per GPU.  Every
rank opens its partition of the same weighted graph, the weighted SSSP exchanges frontiers by NCCL or by P2P pushes, the
per-class sigma pieces are broadcast and the delta partials all-reduced through the communicator.  Cases: an RMAT-16
sample with generator weights against the weighted oracle (rtol 1e-10), the exact weighted forest (bitwise: all-reduce
sums of these values are exact), and a graph whose last partition has no edges (asserted)."""
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
import bc_weighted_oracle as B  # noqa: E402
import weighted_oracle as WO  # noqa: E402
from graphs import trailing_isolated  # noqa: E402


def close(a, b, rtol=1e-10):
    return bool(np.all((a == 0) == (b == 0)) and np.allclose(a, b, rtol=rtol, atol=0))


def edge_free_case(world):
    """trailing_isolated with extra in-edges into the last core vertex (499), as few as make the reference split put every
    edge into the first world - 1 partitions: the last rank holds vertices but no edges."""
    re0, src0 = trailing_isolated()
    nv = len(re0)
    dst0 = np.repeat(np.arange(nv), np.diff(np.concatenate([[0], re0]).astype(np.int64)))
    for k in range(250, 40001, 250):
        row_end, src = O.edges_to_csc(nv, np.concatenate([src0, np.arange(k) % 499]), np.concatenate([dst0, np.full(k, 499)]))
        _, rl, rr, cl = L.partition_csc(row_end, len(src), world)
        if int(cl[-1]) == len(src) and rl[-1] < nv and rr[-1] == nv - 1:
            return row_end, src
    raise AssertionError("no edge-free last partition found for world %d" % world)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    cases = []
    re16, src16 = O.gen_rmat_csc(16, 1 << 16, 16 << 16, 27)
    cases.append(("rmat16", re16, src16, WO.rmat_weights(27, re16, src16),
                  np.random.default_rng(16).choice(1 << 16, 8, replace=False).astype(np.uint32), False))
    f = B.forest()
    cases.append(("forest", f["row_end"], f["src"], f["weight"], f["roots"], True))
    re_t, src_t = edge_free_case(world)
    w_t = np.random.default_rng(5).integers(1, 256, len(src_t)).astype(np.int32)
    cases.append(("edge_free_last_rank", re_t, src_t, w_t, np.array([0, 3, 17, 499, len(re_t) - 1], np.uint32), False))
    ok = True
    for name, row_end, src, w, sources, exact in cases:
        ref = B.run(row_end, src, w, sources)
        for exchange, ename in ((L.EXCHANGE_NCCL, "nccl"), (L.EXCHANGE_P2P, "p2p push")):
            g = L.LuxGraph.from_csc(row_end, src, w, app=L.APP_BC_WEIGHTED, rank=rank, nranks=world, device=local, exchange=exchange)
            g.comm_init_torch()
            g.init()
            connected = exchange == L.EXCHANGE_NCCL or g.p2p_connect_torch()
            g.bc_run(sources)
            bc = g.values()
            lev, sigma, delta = g.bc_source_state()
            b = g.bounds()
            edge_free = int(b["col_left"][-1]) == len(src) and int(b["row_right"][-1]) >= int(b["row_left"][-1])
            if exact:
                good = np.array_equal(bc, f["scores"]) and np.array_equal(delta, ref["delta"])
            else:
                good = close(bc, ref["scores"]) and close(delta, ref["delta"])
            good = connected and good and np.array_equal(lev, ref["dist"]) and np.array_equal(sigma, ref["sigma"])
            if name == "edge_free_last_rank":
                good = good and edge_free
            if rank == 0:
                print("weighted bc [%s, %s] world=%d: %s%s" % (name, ename, world, "OK" if good else "FAIL",
                                                     " (last partition edge-free)" if edge_free else ""), flush=True)
            ok = ok and good
            g.close()
            dist.barrier()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("MGPU_BC_WEIGHTED %s" % ("PASS" if int(flag) else "FAIL"), flush=True)
    sys.exit(0 if int(flag) else 1)


if __name__ == "__main__":
    main()
