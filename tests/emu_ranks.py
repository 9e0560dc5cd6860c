"""Ranks as host threads of one process on one GPU, exchanging through the in-process NCCL stand-in (tests/fake_nccl.c).

Every handle lives in the same process, so every rank's device buffers are valid in every thread and a collective is
a set of copies between them: the multi-rank paths of the library (partition offsets, grouped broadcasts, all-gathers,
all-reduces) run on a one-GPU machine.  The P2P exchange is not emulated (cudaIpcOpenMemHandle cannot open a handle in
the process that exported it).

run_ranks(world, body) runs body(rank, uid) on `world` threads on device 0; uid(i) is the i-th communicator id, the
same in every thread.  It is called inside a subprocess (emulate(), from a pytest test): the subprocess gets
LUXB_NCCL_LIBRARY and any LUXB_* sweep settings in its environment before libluxb binds NCCL, a wall-clock timeout, and
a failure leaves nothing behind in the test process (nor meets the real NCCL torch may have loaded there).

    python tests/emu_ranks.py <module> <case> <json keyword arguments>

runs <module>.<case>(**kwargs) in such a process, once per world when the arguments hold a list "worlds"."""
import json
import os
import subprocess
import sys
import threading
import traceback

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def run_ranks(world, body, timeout=900):
    """body(rank, uid) on `world` threads; returns the list of results.  Raises AssertionError naming every rank that
    raised, with its message (the bodies' assertions name the case and the first differing index)."""
    import lux_b200 as L
    lock = threading.Lock()
    ids = []

    def uid(i=0):
        with lock:
            while len(ids) <= i:
                ids.append(L.LuxGraph.comm_unique_id())
            return ids[i]

    uid(0)  # binds NCCL in this thread first: the stand-in, or an error
    out, err = [None] * world, [None] * world

    def run(r):
        try:
            out[r] = body(r, uid)
        except BaseException:  # noqa: BLE001
            err[r] = traceback.format_exc()

    threads = [threading.Thread(target=run, args=(r,), daemon=True) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=timeout)
    hung = [r for r, t in enumerate(threads) if t.is_alive()]
    if hung:
        raise AssertionError("world %d: ranks %s did not finish within %d s" % (world, hung, timeout))
    fake = os.environ.get("LUXB_NCCL_LIBRARY", "")
    if world > 1 and all(e is None for e in err):
        with open("/proc/self/maps") as f:
            assert fake and fake in f.read(), "libluxb did not bind the NCCL stand-in (%r)" % fake
    bad = [(r, e) for r, e in enumerate(err) if e is not None]
    if bad:
        raise AssertionError("world %d: %d rank(s) failed\n%s" % (world, len(bad), "\n".join(
            "---- rank %d ----\n%s" % (r, e.strip()[-3000:]) for r, e in bad[:4])))
    return out


def emulate(module, case, env=None, timeout=1200, **kwargs):
    """Run module.case(**kwargs) in a fresh interpreter with the stand-in bound, once per world of kwargs["worlds"] if
    given; returns (exit code, output with stderr merged in order)."""
    import fake_nccl
    e = dict(os.environ)
    e.update({"LUXB_NCCL_LIBRARY": fake_nccl.build(), "PYTHONPATH": os.pathsep.join([ROOT, HERE])})
    e.update({k: str(v) for k, v in (env or {}).items()})
    cmd = [sys.executable, os.path.abspath(__file__), module, case, json.dumps(kwargs)]
    try:
        p = subprocess.run(cmd, cwd=ROOT, env=e, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout)
    except subprocess.TimeoutExpired as t:
        return -1, "timed out after %d s\n%s" % (timeout, (t.output or b"").decode(errors="replace")[-6000:])
    return p.returncode, p.stdout.decode(errors="replace")


def main():
    for p in (ROOT, HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    module, case, kwargs = sys.argv[1], sys.argv[2], json.loads(sys.argv[3])
    mod = __import__(module)
    worlds = kwargs.pop("worlds", None)
    try:
        for w in worlds if worlds is not None else [None]:
            getattr(mod, case)(**kwargs) if w is None else getattr(mod, case)(world=w, **kwargs)
    except BaseException:  # noqa: BLE001
        print("EMULATED CASE FAILED: %s.%s(%s) at world %s" % (module, case, kwargs, w), flush=True)
        traceback.print_exc()
        sys.stdout.flush()
        os._exit(1)  # without joining daemon rank threads that may still wait
    print("EMULATED CASE PASSED: %s.%s(%s) at worlds %s" % (module, case, kwargs, worlds), flush=True)
    sys.stdout.flush()
    os._exit(0)


if __name__ == "__main__":
    main()
