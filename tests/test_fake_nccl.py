"""CPU: the in-process NCCL stand-in (tests/fake_nccl.c) on host buffers (FAKE_NCCL_HOST=1), driven by one thread per
rank through ctypes.  It pins what the emulated-rank GPU tests rely on, so that a failure there points at the library and
not at the stand-in:
  * broadcast from every root, all-gather and all-reduce, out of place and in place, for every data type libluxb passes
    (broadcast u8 / u32 / u64 / f32 / f64, all-reduce sums of u8 / u32 / u64 / f64, the f64 sum taken in rank order);
  * the all-gather whose send buffer lies inside the receive allocation (TC's count exchange), a root whose send buffer
    differs from its receive buffer inside a group (TC's key exchange);
  * grouped broadcasts with a different root per call (the PageRank / frontier exchanges), nested groups;
  * other types and ops rejected; a mismatched call sequence reported on every rank with the rank and the call named;
  * a rank that never joins or never calls: the others get a timeout error, not a hang;
  * worlds of 1, 3 and 64 ranks; unique ids."""
import ctypes as C
import threading

import numpy as np
import pytest

import fake_nccl as F

DTYPES = {F.UINT8: np.uint8, F.UINT32: np.uint32, F.UINT64: np.uint64, F.FLOAT32: np.float32, F.FLOAT64: np.float64}
REDUCE_DTYPES = (F.UINT8, F.UINT32, F.UINT64, F.FLOAT64)
WORLDS = [1, 3, 64]


@pytest.fixture(autouse=True)
def host_mode(monkeypatch):
    monkeypatch.setenv("FAKE_NCCL_HOST", "1")
    monkeypatch.setenv("FAKE_NCCL_TIMEOUT_S", "30")


def _ptr(a, offset=0):
    return C.c_void_p(a.ctypes.data + int(offset) * a.itemsize)


class Rank:
    """One rank's communicator; every call returns (rc, message) read in the calling thread."""

    def __init__(self, comm, rank, P):
        self.comm, self.rank, self.P = comm, rank, P

    def _rc(self, rc):
        return rc, (F.lib().ncclGetErrorString(rc).decode() if rc else "")

    def bcast(self, send, recv, count, dtype, root):
        return self._rc(F.lib().ncclBroadcast(send, recv, count, dtype, root, self.comm, None))

    def gather(self, send, recv, count, dtype):
        return self._rc(F.lib().ncclAllGather(send, recv, count, dtype, self.comm, None))

    def reduce(self, send, recv, count, dtype, op=F.SUM):
        return self._rc(F.lib().ncclAllReduce(send, recv, count, dtype, op, self.comm, None))

    def group_start(self):
        assert F.lib().ncclGroupStart() == 0

    def group_end(self):
        return self._rc(F.lib().ncclGroupEnd())


def new_id():
    uid = F.UniqueId()
    assert F.lib().ncclGetUniqueId(C.byref(uid)) == 0
    return uid


def run_world(P, body, ranks=None, uid=None):
    """body(Rank) on P threads (only `ranks` of them join when given); returns the bodies' results, raises the first
    exception with its rank."""
    uid = new_id() if uid is None else uid
    out, err = [None] * P, [None] * P

    def run(r):
        try:
            comm = C.c_void_p()
            rc = F.lib().ncclCommInitRank(C.byref(comm), P, uid, r)
            if rc:
                out[r] = ("init", rc, F.lib().ncclGetErrorString(rc).decode())
                return
            try:
                out[r] = body(Rank(comm, r, P))
            finally:
                F.lib().ncclCommDestroy(comm)
        except BaseException as e:  # noqa: BLE001
            err[r] = e

    threads = [threading.Thread(target=run, args=(r,)) for r in (range(P) if ranks is None else ranks)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=120)
        assert not t.is_alive(), "a rank thread did not finish"
    for r, e in enumerate(err):
        if e is not None:
            raise AssertionError("rank %d: %r" % (r, e)) from e
    return out


def values(dtype, n, seed):
    rng = np.random.default_rng(seed)
    if np.dtype(dtype).kind == "f":
        return (rng.standard_normal(n) * 10.0 ** rng.integers(-8, 8, n)).astype(dtype)
    return rng.integers(0, np.iinfo(dtype).max, n, dtype=dtype, endpoint=True)


# ---- single collectives ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", sorted(DTYPES))
def test_broadcast_every_root_in_and_out_of_place(P, dtype):
    n = 37
    npt = DTYPES[dtype]
    src = [values(npt, n, 100 * r + dtype) for r in range(P)]

    def body(k):
        got = []
        for root in range(P):
            send = src[k.rank].copy()
            recv = values(npt, n, 7)  # garbage that must be overwritten
            assert k.bcast(_ptr(send), _ptr(recv), n, dtype, root) == (0, "")
            inplace = src[k.rank].copy()
            assert k.bcast(_ptr(inplace), _ptr(inplace), n, dtype, root) == (0, "")
            assert np.array_equal(send, src[k.rank])  # a send buffer is never written
            got.append((recv, inplace))
        return got

    for r, got in enumerate(run_world(P, body)):
        for root, (recv, inplace) in enumerate(got):
            assert np.array_equal(recv, src[root]), (r, root)
            assert np.array_equal(inplace, src[root]), (r, root)


@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", [F.UINT8, F.UINT64, F.FLOAT32])
def test_allgather_out_of_place_in_place_and_send_inside_recv(P, dtype):
    n = 5
    npt = DTYPES[dtype]
    src = [values(npt, n, 10 * r + dtype) for r in range(P)]
    want = np.concatenate(src)

    def body(k):
        recv = np.zeros(P * n, npt)
        assert k.gather(_ptr(src[k.rank]), _ptr(recv), n, dtype) == (0, "")
        inplace = np.zeros(P * n, npt)  # NCCL's in-place form: send = recv + rank * count
        inplace[k.rank * n:(k.rank + 1) * n] = src[k.rank]
        assert k.gather(_ptr(inplace, k.rank * n), _ptr(inplace), n, dtype) == (0, "")
        tail = np.zeros((P + 1) * n, npt)  # send just past the receive range of the same allocation
        tail[P * n:] = src[k.rank]
        assert k.gather(_ptr(tail, P * n), _ptr(tail), n, dtype) == (0, "")
        return recv, inplace, tail

    for r, (recv, inplace, tail) in enumerate(run_world(P, body)):
        assert np.array_equal(recv, want), r
        assert np.array_equal(inplace, want), r
        assert np.array_equal(tail[:P * n], want) and np.array_equal(tail[P * n:], src[r]), r


@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", REDUCE_DTYPES)
def test_allreduce_sums_in_rank_order(P, dtype):
    n = 101
    npt = DTYPES[dtype]
    src = [values(npt, n, 1000 + r) for r in range(P)]
    want = src[0].copy()
    with np.errstate(over="ignore"):
        for r in range(1, P):  # integers wrap; floats are summed rank after rank
            want = (want + src[r]).astype(npt)

    def body(k):
        recv = np.zeros(n, npt)
        assert k.reduce(_ptr(src[k.rank]), _ptr(recv), n, dtype) == (0, "")
        inplace = src[k.rank].copy()
        assert k.reduce(_ptr(inplace), _ptr(inplace), n, dtype) == (0, "")
        return recv, inplace

    for r, (recv, inplace) in enumerate(run_world(P, body)):
        assert np.array_equal(recv.view(np.uint8), want.view(np.uint8)), r
        assert np.array_equal(inplace.view(np.uint8), want.view(np.uint8)), r
    if dtype == F.FLOAT64 and P == 64:
        assert not np.array_equal(want, np.sum(np.stack(src[::-1]), axis=0)), "inputs do not tell one order from another"


def test_unsupported_types_and_ops_are_errors():
    def body(k):
        a = np.zeros(4, np.float32)
        b = np.zeros(4, np.uint32)
        return [k.reduce(_ptr(a), _ptr(a), 4, F.FLOAT32), k.reduce(_ptr(b), _ptr(b), 4, F.UINT32, op=F.PROD),
                k.reduce(_ptr(b), _ptr(b), 4, F.INT32), k.bcast(_ptr(b), _ptr(b), 4, 42, 0), k.bcast(_ptr(b), _ptr(b), 4, F.UINT32, 3),
                k.reduce(_ptr(b), _ptr(b), 4, F.UINT32)]

    for out in run_world(2, body):
        for rc, msg in out[:5]:
            assert rc == F.INVALID_ARGUMENT and msg.startswith("fake NCCL"), (rc, msg)
        assert out[5] == (0, "")  # the communicator still works


# ---- groups ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", WORLDS)
def test_grouped_broadcasts_with_every_root(P):
    """Every rank owns a ragged slice of one replicated array and broadcasts it in place, all P broadcasts in one group
    (PageRank's packed ranges, the frontier slots); then a nested group where each root sends from a private buffer into
    the shared array (TC's key exchange)."""
    sizes = [(3 * p) % 7 for p in range(P)]  # some slices are empty
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(int)
    full = values(np.uint32, int(off[-1]), 3)

    def body(k):
        rep = np.zeros(len(full), np.uint32)
        rep[off[k.rank]:off[k.rank + 1]] = full[off[k.rank]:off[k.rank + 1]]
        k.group_start()
        for p in range(P):
            if sizes[p]:
                seg = _ptr(rep, off[p])
                assert k.bcast(seg, seg, sizes[p] * 4, F.UINT8, p) == (0, "")
        assert k.group_end() == (0, "")
        mine = full[off[k.rank]:off[k.rank + 1]].copy()
        rep2 = np.zeros(len(full), np.uint32)
        k.group_start()
        k.group_start()
        for p in range(P):
            if sizes[p]:
                send = _ptr(mine) if p == k.rank else _ptr(rep2, off[p])
                assert k.bcast(send, _ptr(rep2, off[p]), sizes[p], F.UINT32, p) == (0, "")
        assert k.group_end() == (0, "")  # inner: nothing runs yet
        assert k.group_end() == (0, "")
        return rep, rep2

    for r, (rep, rep2) in enumerate(run_world(P, body)):
        assert np.array_equal(rep, full), r
        assert np.array_equal(rep2, full), r


# ---- protocol errors ---------------------------------------------------------------------------------------------------
def test_mismatched_sequence_is_reported_on_every_rank():
    P = 3

    def body(k):
        a = np.zeros(16, np.uint32)
        out = [k.bcast(_ptr(a), _ptr(a), 8 if k.rank != 2 else 9, F.UINT32, 0)]
        k.group_start()  # rank 1 leaves out the second broadcast of the group
        k.bcast(_ptr(a), _ptr(a), 4, F.UINT32, 0)
        if k.rank != 1:
            k.bcast(_ptr(a), _ptr(a), 4, F.UINT32, 2)
        out.append(k.group_end())
        out.append(k.reduce(_ptr(a), _ptr(a), 16, F.UINT32))  # in step again
        return out

    for r, out in enumerate(run_world(P, body)):
        (rc0, m0), (rc1, m1), ok = out
        assert rc0 == F.INVALID_USAGE and "rank 2 issued ncclBroadcast(count 9" in m0 and "call 0" in m0, (r, m0)
        assert rc1 == F.INVALID_USAGE and "rank 1 issued nothing" in m1 and "call 1" in m1, (r, m1)
        assert ok == (0, ""), (r, ok)


def test_missing_rank_times_out_at_init(monkeypatch):
    monkeypatch.setenv("FAKE_NCCL_TIMEOUT_S", "1")
    out = run_world(3, lambda k: None, ranks=[0, 1])
    for r in (0, 1):
        kind, rc, msg = out[r]
        assert kind == "init" and rc == F.SYSTEM_ERROR and "only 2 of 3 ranks joined" in msg, out[r]


def test_missing_rank_times_out_in_a_collective(monkeypatch):
    monkeypatch.setenv("FAKE_NCCL_TIMEOUT_S", "1")

    def body(k):
        a = np.zeros(4, np.uint64)
        if k.rank == 2:
            return None  # joins, then never calls
        return k.reduce(_ptr(a), _ptr(a), 4, F.UINT64), k.reduce(_ptr(a), _ptr(a), 4, F.UINT64)

    out = run_world(3, body)
    for r in (0, 1):
        (rc, msg), (rc2, msg2) = out[r]
        assert rc == F.SYSTEM_ERROR and "timed out" in msg and "barrier 1" in msg, msg
        assert rc2 == F.SYSTEM_ERROR and "timed out" in msg2, msg2  # broken: later calls fail at once


def test_unique_ids_and_init_arguments(monkeypatch):
    ids = {bytes(new_id().internal) for _ in range(1000)}
    assert len(ids) == 1000
    monkeypatch.setenv("FAKE_NCCL_TIMEOUT_S", "1")
    uid = new_id()
    out = [None, None]

    def join(r, P):
        comm = C.c_void_p()
        rc = F.lib().ncclCommInitRank(C.byref(comm), P, uid, r)
        out[r] = (rc, F.lib().ncclGetErrorString(rc).decode() if rc else "")

    t = threading.Thread(target=join, args=(0, 2))
    t.start()
    join(1, 3)  # the same id with another world size: whichever rank comes second is refused, the first one times out
    t.join(timeout=60)
    assert sorted(rc for rc, _ in out) == [F.SYSTEM_ERROR, F.INVALID_USAGE], out
    assert any("joins with nranks" in m for _, m in out) and any("only 1 of" in m for _, m in out), out
    comm = C.c_void_p()
    assert F.lib().ncclCommInitRank(C.byref(comm), 2, new_id(), 2) == F.INVALID_ARGUMENT
