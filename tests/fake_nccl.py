"""Build and bind tests/fake_nccl.c, the in-process NCCL stand-in for ranks that are threads of one process on one
device (test infrastructure only).  libluxb loads it when LUXB_NCCL_LIBRARY names it (tests/emu_ranks.py);
tests/test_fake_nccl.py drives it directly through ctypes on host buffers (FAKE_NCCL_HOST=1).

The library is compiled with gcc on first use into a per-user cache directory keyed by the digest of the C source (the
source tree is never written)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fake_nccl.c")
_CFLAGS = ["-O2", "-fPIC", "-pthread", "-Wall", "-Wextra", "-std=gnu11", "-shared"]
_lib = None

# nccl.h values
INT8, UINT8, INT32, UINT32, INT64, UINT64, FLOAT16, FLOAT32, FLOAT64 = 0, 1, 2, 3, 4, 5, 6, 7, 8
SUM, PROD = 0, 1
SUCCESS, INVALID_ARGUMENT, INVALID_USAGE, SYSTEM_ERROR = 0, 4, 5, 2


class UniqueId(C.Structure):
    _fields_ = [("internal", C.c_char * 128)]  # passed by value, like ncclUniqueId


def build():
    """Path of the compiled library, building it if this digest of the source has not been built yet."""
    with open(_SRC, "rb") as f:
        digest = hashlib.sha256(f.read() + " ".join(_CFLAGS).encode()).hexdigest()[:16]
    cache = os.path.join(tempfile.gettempdir(), "luxb_fake_nccl_%d" % os.getuid())
    os.makedirs(cache, exist_ok=True)
    so = os.path.join(cache, "libfake_nccl_%s.so" % digest)
    if not os.path.exists(so):
        tmp = "%s.tmp.%d" % (so, os.getpid())
        subprocess.check_call(["gcc"] + _CFLAGS + ["-o", tmp, _SRC, "-ldl"])
        os.replace(tmp, so)  # atomic: concurrent builders never load a half-written library
    return so


def lib():
    """The fake bound through ctypes (its own handle; libluxb binds it separately through dlopen)."""
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        vp, sz = C.c_void_p, C.c_size_t
        for name, args in (("ncclGetUniqueId", [vp]), ("ncclCommInitRank", [vp, C.c_int, UniqueId, C.c_int]),
                           ("ncclCommDestroy", [vp]), ("ncclAllReduce", [vp, vp, sz, C.c_int, C.c_int, vp, vp]),
                           ("ncclBroadcast", [vp, vp, sz, C.c_int, C.c_int, vp, vp]),
                           ("ncclAllGather", [vp, vp, sz, C.c_int, vp, vp]), ("ncclGroupStart", []), ("ncclGroupEnd", [])):
            f = getattr(L, name)
            f.argtypes, f.restype = args, C.c_int
        L.ncclGetErrorString.argtypes, L.ncclGetErrorString.restype = [C.c_int], C.c_char_p
        _lib = L
    return _lib
