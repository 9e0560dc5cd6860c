// fake_nccl.c — an in-process stand-in for the nine NCCL entry points libluxb binds at run time (lux_b200/csrc/comm.h),
// for ranks that are host threads of ONE process sharing one device.  Loaded through LUXB_NCCL_LIBRARY by the emulated-rank
// tests (tests/emu_ranks.py); test infrastructure only, never part of the library.
//
// Every handle lives in the same process, so every rank's device pointer is valid in every thread, and a collective is a
// set of copies between the ranks' buffers.  Each step (one collective, or one group of them) runs in two phases, which
// makes every aliasing safe (in-place broadcast, AllGather(send inside recv), a root whose send differs from its recv):
//   1. synchronise the caller's stream, publish this rank's operations, wait at barrier 1; check that every rank issued
//      the same (kind, count, dtype, op, root) sequence; read what this rank needs from the peers' send buffers into
//      private host staging (all-reduce: summed in rank order);
//   2. wait at barrier 2, then write this rank's own receive buffers from the staging and synchronise the stream.
// A mismatched sequence is an error on every rank (real NCCL would hang or corrupt data), and its message, returned by
// ncclGetErrorString in the failing thread, names the rank and the call.  Every wait has a host-side timeout
// (FAKE_NCCL_TIMEOUT_S, default 120 s): a rank that never arrives turns into errors on the others, not a hung process.
// Nothing spins on the device.
//
// Device mode reaches memory through the driver API (libcuda.so.1, dlopen'ed: no second cudart in the process), on the
// caller's stream and in the caller's current context.  FAKE_NCCL_HOST=1 (read at ncclCommInitRank) makes every buffer a
// host buffer copied with memcpy, so the semantics can be tested without a GPU.
#define _GNU_SOURCE
#include <dlfcn.h>
#include <errno.h>
#include <pthread.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>

typedef enum {
  ncclSuccess = 0,
  ncclUnhandledCudaError = 1,
  ncclSystemError = 2,
  ncclInternalError = 3,
  ncclInvalidArgument = 4,
  ncclInvalidUsage = 5
} ncclResult_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { ncclUint8 = 1, ncclUint32 = 3, ncclUint64 = 5, ncclFloat64 = 8, ncclNumTypes = 10 };
enum { ncclSum = 0 };
enum { KIND_BROADCAST, KIND_ALLGATHER, KIND_ALLREDUCE };
static const char* const KIND_NAME[] = {"ncclBroadcast", "ncclAllGather", "ncclAllReduce"};
// bytes per element of ncclInt8 .. ncclBfloat16 (nccl.h)
static const size_t TYPE_BYTES[ncclNumTypes] = {1, 1, 4, 4, 8, 8, 2, 4, 8, 2};

// ---- driver API, bound at first use ----------------------------------------------------------------------------------
typedef int CUresult;
typedef unsigned long long CUdeviceptr;
static struct {
  pthread_once_t once;
  const char* err;
  CUresult (*dtoh)(void*, CUdeviceptr, size_t, void*);
  CUresult (*htod)(CUdeviceptr, const void*, size_t, void*);
  CUresult (*sync)(void*);
  CUresult (*ctx_current)(void**);
} cu = {PTHREAD_ONCE_INIT, NULL, NULL, NULL, NULL, NULL};

static void cu_load(void) {
  void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_LOCAL);
  if (!h) {
    cu.err = "cannot dlopen libcuda.so.1";
    return;
  }
  cu.dtoh = (CUresult(*)(void*, CUdeviceptr, size_t, void*))dlsym(h, "cuMemcpyDtoHAsync_v2");
  cu.htod = (CUresult(*)(CUdeviceptr, const void*, size_t, void*))dlsym(h, "cuMemcpyHtoDAsync_v2");
  cu.sync = (CUresult(*)(void*))dlsym(h, "cuStreamSynchronize");
  cu.ctx_current = (CUresult(*)(void**))dlsym(h, "cuCtxGetCurrent");
  if (!cu.dtoh || !cu.htod || !cu.sync || !cu.ctx_current) cu.err = "libcuda.so.1 lacks a driver entry point";
}

// ---- errors: the message of the last failure in this thread ------------------------------------------------------------
static __thread char t_err[1024];

static ncclResult_t fail(ncclResult_t rc, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  int n = snprintf(t_err, sizeof t_err, "fake NCCL: ");
  vsnprintf(t_err + n, sizeof t_err - n, fmt, ap);
  va_end(ap);
  return rc;
}

const char* ncclGetErrorString(ncclResult_t rc) {
  if (t_err[0]) return t_err;
  return rc == ncclSuccess ? "no error" : "fake NCCL: error";
}

// ---- communicators -----------------------------------------------------------------------------------------------------
typedef struct {
  int kind, dtype, op, root;
  size_t count;
  const void* send;
  void* recv;
  void* stream;
  size_t stage_off;  // this op's place in the rank's staging buffer
} Op;

typedef struct Shared {
  ncclUniqueId id;
  int nranks, joined, refs, host;
  double timeout_s;
  pthread_mutex_t mu;
  pthread_cond_t cv;
  unsigned long gen;  // barrier generation
  int arrived;
  int broken;  // a rank timed out: every later wait fails at once
  char why[512];
  const Op** ops;  // ops[r]: the step rank r published before barrier 1 (read only in phase 1)
  int* nops;
  struct Shared* next;
} Shared;

struct ncclComm {
  Shared* s;
  int rank;
  unsigned long steps;
};
typedef struct ncclComm* ncclComm_t;

static pthread_mutex_t g_registry_mu = PTHREAD_MUTEX_INITIALIZER;
static Shared* g_registry;  // communicators whose ranks have not all joined yet
static unsigned long g_next_id;

static double env_timeout(void) {
  const char* t = getenv("FAKE_NCCL_TIMEOUT_S");
  double v = t ? atof(t) : 0.0;
  return v > 0 ? v : 120.0;
}

static struct timespec deadline(double s) {
  struct timespec ts;
  clock_gettime(CLOCK_REALTIME, &ts);
  time_t whole = (time_t)s;
  long ns = ts.tv_nsec + (long)((s - (double)whole) * 1e9);
  ts.tv_sec += whole + ns / 1000000000L;
  ts.tv_nsec = ns % 1000000000L;
  return ts;
}

ncclResult_t ncclGetUniqueId(ncclUniqueId* id) {
  if (!id) return fail(ncclInvalidArgument, "ncclGetUniqueId: null id");
  memset(id, 0, sizeof *id);
  pthread_mutex_lock(&g_registry_mu);
  unsigned long n = ++g_next_id;
  pthread_mutex_unlock(&g_registry_mu);
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  snprintf(id->internal, sizeof id->internal, "fake-nccl pid %ld id %lu t %ld.%09ld", (long)getpid(), n, (long)ts.tv_sec, ts.tv_nsec);
  return ncclSuccess;
}

ncclResult_t ncclCommInitRank(ncclComm_t* comm, int nranks, ncclUniqueId id, int rank) {
  if (!comm || nranks < 1 || rank < 0 || rank >= nranks)
    return fail(ncclInvalidArgument, "ncclCommInitRank: rank %d of %d", rank, nranks);
  const char* host = getenv("FAKE_NCCL_HOST");
  int host_mode = host && strcmp(host, "1") == 0;
  if (!host_mode) {
    pthread_once(&cu.once, cu_load);
    if (cu.err) return fail(ncclUnhandledCudaError, "%s", cu.err);
  }
  pthread_mutex_lock(&g_registry_mu);
  Shared* s = g_registry;
  while (s && memcmp(s->id.internal, id.internal, sizeof id.internal) != 0) s = s->next;
  if (!s) {
    s = (Shared*)calloc(1, sizeof *s);
    if (!s) {
      pthread_mutex_unlock(&g_registry_mu);
      return fail(ncclSystemError, "out of host memory");
    }
    s->id = id;
    s->nranks = nranks;
    s->host = host_mode;
    s->timeout_s = env_timeout();
    pthread_mutex_init(&s->mu, NULL);
    pthread_cond_init(&s->cv, NULL);
    s->ops = (const Op**)calloc(nranks, sizeof *s->ops);
    s->nops = (int*)calloc(nranks, sizeof *s->nops);
    s->next = g_registry;
    g_registry = s;
  }
  pthread_mutex_lock(&s->mu);
  if (s->nranks != nranks || s->host != host_mode) {
    pthread_mutex_unlock(&s->mu);
    pthread_mutex_unlock(&g_registry_mu);
    return fail(ncclInvalidUsage, "ncclCommInitRank: rank %d joins with nranks %d (host mode %d), the communicator has %d (%d)",
                rank, nranks, host_mode, s->nranks, s->host);
  }
  s->joined++;
  s->refs++;
  if (s->joined == s->nranks) {  // complete: later ids never match it
    Shared** pp = &g_registry;
    while (*pp != s) pp = &(*pp)->next;
    *pp = s->next;
    pthread_cond_broadcast(&s->cv);
  }
  pthread_mutex_unlock(&g_registry_mu);
  struct timespec until = deadline(s->timeout_s);
  int rc = 0;
  while (s->joined < s->nranks && !s->broken && rc != ETIMEDOUT) rc = pthread_cond_timedwait(&s->cv, &s->mu, &until);
  if (s->joined < s->nranks) {
    // the communicator stays allocated: ranks that join late find it broken
    if (!s->broken) {
      s->broken = 1;
      snprintf(s->why, sizeof s->why, "ncclCommInitRank: only %d of %d ranks joined within %.0f s", s->joined, s->nranks, s->timeout_s);
      pthread_cond_broadcast(&s->cv);
    }
    pthread_mutex_unlock(&s->mu);
    return fail(ncclSystemError, "rank %d: %s", rank, s->why);
  }
  pthread_mutex_unlock(&s->mu);
  struct ncclComm* c = (struct ncclComm*)calloc(1, sizeof *c);
  if (!c) return fail(ncclSystemError, "out of host memory");
  c->s = s;
  c->rank = rank;
  *comm = c;
  return ncclSuccess;
}

ncclResult_t ncclCommDestroy(ncclComm_t comm) {
  if (!comm) return ncclSuccess;
  Shared* s = comm->s;
  pthread_mutex_lock(&s->mu);
  int last = --s->refs == 0;
  pthread_mutex_unlock(&s->mu);
  free(comm);
  if (last) {
    pthread_mutex_destroy(&s->mu);
    pthread_cond_destroy(&s->cv);
    free(s->ops);
    free(s->nops);
    free(s);
  }
  return ncclSuccess;
}

// wait until every rank of the communicator has arrived; fails on timeout, or when another rank timed out before
static ncclResult_t barrier(struct ncclComm* c, const char* where) {
  Shared* s = c->s;
  pthread_mutex_lock(&s->mu);
  if (s->broken) {
    pthread_mutex_unlock(&s->mu);
    return fail(ncclSystemError, "rank %d, step %lu (%s): %s", c->rank, c->steps, where, s->why);
  }
  unsigned long gen = s->gen;
  if (++s->arrived == s->nranks) {
    s->arrived = 0;
    s->gen++;
    pthread_cond_broadcast(&s->cv);
    pthread_mutex_unlock(&s->mu);
    return ncclSuccess;
  }
  struct timespec until = deadline(s->timeout_s);
  int rc = 0;
  while (s->gen == gen && !s->broken && rc != ETIMEDOUT) rc = pthread_cond_timedwait(&s->cv, &s->mu, &until);
  if (s->gen == gen) {
    if (!s->broken) {
      s->broken = 1;
      snprintf(s->why, sizeof s->why, "rank %d timed out after %.0f s at %s with %d of %d ranks arrived", c->rank, s->timeout_s,
               where, s->arrived, s->nranks);
      pthread_cond_broadcast(&s->cv);
    }
    pthread_mutex_unlock(&s->mu);
    return fail(ncclSystemError, "rank %d, step %lu (%s): %s", c->rank, c->steps, where, s->why);
  }
  pthread_mutex_unlock(&s->mu);
  return ncclSuccess;
}

// ---- copies ------------------------------------------------------------------------------------------------------------
static ncclResult_t read_buf(struct ncclComm* c, void* stage, const void* src, size_t bytes, void* stream) {
  if (!bytes) return ncclSuccess;
  if (c->s->host) {
    memcpy(stage, src, bytes);
    return ncclSuccess;
  }
  CUresult r = cu.dtoh(stage, (CUdeviceptr)(uintptr_t)src, bytes, stream);
  if (!r) r = cu.sync(stream);
  return r ? fail(ncclUnhandledCudaError, "rank %d: device-to-host copy of %zu bytes from %p failed (CUresult %d)", c->rank, bytes,
                  src, r)
           : ncclSuccess;
}

static ncclResult_t write_buf(struct ncclComm* c, void* dst, const void* stage, size_t bytes, void* stream) {
  if (!bytes) return ncclSuccess;
  if (c->s->host) {
    memcpy(dst, stage, bytes);
    return ncclSuccess;
  }
  CUresult r = cu.htod((CUdeviceptr)(uintptr_t)dst, stage, bytes, stream);
  return r ? fail(ncclUnhandledCudaError, "rank %d: host-to-device copy of %zu bytes to %p failed (CUresult %d)", c->rank, bytes,
                  dst, r)
           : ncclSuccess;
}

static void add_into(void* acc, const void* x, size_t n, int dtype) {
  size_t i;
  switch (dtype) {
    case ncclUint8:
      for (i = 0; i < n; i++) ((uint8_t*)acc)[i] = (uint8_t)(((uint8_t*)acc)[i] + ((const uint8_t*)x)[i]);
      break;
    case ncclUint32:
      for (i = 0; i < n; i++) ((uint32_t*)acc)[i] += ((const uint32_t*)x)[i];
      break;
    case ncclUint64:
      for (i = 0; i < n; i++) ((uint64_t*)acc)[i] += ((const uint64_t*)x)[i];
      break;
    case ncclFloat64:
      for (i = 0; i < n; i++) ((double*)acc)[i] += ((const double*)x)[i];
      break;
  }
}

static size_t recv_bytes(const Op* o, int nranks) {
  size_t b = o->count * TYPE_BYTES[o->dtype];
  return o->kind == KIND_ALLGATHER ? b * (size_t)nranks : b;
}

// ---- steps: one collective, or one group ---------------------------------------------------------------------------------
static __thread struct {
  int depth;
  int failed;  // an operation of the open group was rejected: its GroupEnd runs nothing and fails
  struct ncclComm* comm;
  Op* ops;
  int n, cap;
  char* stage;
  size_t stage_cap;
  void* tmp;
  size_t tmp_cap;
} t_grp;

static int grow(void** p, size_t* cap, size_t need) {
  if (need <= *cap) return 1;
  void* q = realloc(*p, need);
  if (!q) return 0;
  *p = q;
  *cap = need;
  return 1;
}

static void describe(char* out, size_t n, const Op* o) {
  snprintf(out, n, "%s(count %zu, dtype %d, op %d, root %d)", KIND_NAME[o->kind], o->count, o->dtype, o->op, o->root);
}

static ncclResult_t run_step(struct ncclComm* c, Op* ops, int n) {
  Shared* s = c->s;
  const int P = s->nranks, me = c->rank;
  ncclResult_t rc = ncclSuccess;
  size_t total = 0;
  for (int i = 0; i < n; i++) {
    ops[i].stage_off = total;
    total += (recv_bytes(&ops[i], P) + 15) & ~(size_t)15;
  }
  if (!grow((void**)&t_grp.stage, &t_grp.stage_cap, total ? total : 1)) return fail(ncclSystemError, "out of host memory");
  if (!s->host) {
    void* ctx = NULL;
    if (cu.ctx_current(&ctx) || !ctx) return fail(ncclUnhandledCudaError, "rank %d: no current CUDA context in this thread", me);
    for (int i = 0; i < n; i++) {  // the rank's kernels that produce its send buffers have finished
      CUresult r = cu.sync(ops[i].stream);
      if (r) return fail(ncclUnhandledCudaError, "rank %d: cuStreamSynchronize failed (CUresult %d)", me, r);
    }
  }
  s->ops[me] = ops;
  s->nops[me] = n;
  ncclResult_t b = barrier(c, "barrier 1");
  if (b) return b;
  // phase 1: every rank checks the same published sequences, so all of them agree on a mismatch
  for (int r = 1; r < P && rc == ncclSuccess; r++) {
    const Op* a = s->ops[0];
    const Op* o = s->ops[r];
    int m = s->nops[r] < s->nops[0] ? s->nops[r] : s->nops[0];
    for (int i = 0; i <= m && rc == ncclSuccess; i++) {
      char da[160] = "nothing", dr[160] = "nothing";
      if (i == m) {
        if (s->nops[r] == s->nops[0]) break;
        if (i < s->nops[0]) describe(da, sizeof da, &a[i]);
        if (i < s->nops[r]) describe(dr, sizeof dr, &o[i]);
      } else if (a[i].kind != o[i].kind || a[i].count != o[i].count || a[i].dtype != o[i].dtype || a[i].op != o[i].op ||
                 a[i].root != o[i].root) {
        describe(da, sizeof da, &a[i]);
        describe(dr, sizeof dr, &o[i]);
      } else {
        continue;
      }
      rc = fail(ncclInvalidUsage, "step %lu, call %d of %d: rank %d issued %s where rank 0 issued %s (seen by rank %d)", c->steps, i,
                s->nops[r], r, dr, da, me);
    }
  }
  for (int i = 0; i < n && rc == ncclSuccess; i++) {
    const Op* o = &ops[i];
    char* st = t_grp.stage + o->stage_off;
    size_t bytes = o->count * TYPE_BYTES[o->dtype];
    if (o->kind == KIND_BROADCAST) {
      rc = read_buf(c, st, s->ops[o->root][i].send, bytes, o->stream);
    } else if (o->kind == KIND_ALLGATHER) {
      for (int r = 0; r < P && rc == ncclSuccess; r++) rc = read_buf(c, st + (size_t)r * bytes, s->ops[r][i].send, bytes, o->stream);
    } else {
      rc = read_buf(c, st, s->ops[0][i].send, bytes, o->stream);
      if (P > 1 && !grow(&t_grp.tmp, &t_grp.tmp_cap, bytes)) rc = fail(ncclSystemError, "out of host memory");
      for (int r = 1; r < P && rc == ncclSuccess; r++) {  // rank order, one rank at a time
        rc = read_buf(c, t_grp.tmp, s->ops[r][i].send, bytes, o->stream);
        if (rc == ncclSuccess) add_into(st, t_grp.tmp, o->count, o->dtype);
      }
    }
  }
  b = barrier(c, "barrier 2");
  if (rc == ncclSuccess) rc = b;
  // phase 2: only this rank's own receive buffers
  for (int i = 0; i < n && rc == ncclSuccess; i++)
    rc = write_buf(c, ops[i].recv, t_grp.stage + ops[i].stage_off, recv_bytes(&ops[i], P), ops[i].stream);
  if (!s->host && rc == ncclSuccess) {
    for (int i = 0; i < n && rc == ncclSuccess; i++) {
      CUresult r = cu.sync(ops[i].stream);
      if (r) rc = fail(ncclUnhandledCudaError, "rank %d: cuStreamSynchronize failed (CUresult %d)", me, r);
    }
  }
  c->steps++;
  return rc;
}

static ncclResult_t enqueue(int kind, const void* send, void* recv, size_t count, int dtype, int op, int root, ncclComm_t comm,
                            void* stream) {
  Op o = {kind, dtype, op, root, count, send, recv, stream, 0};
  const char* name = KIND_NAME[kind];
  ncclResult_t rc = ncclSuccess;
  if (!comm)
    rc = fail(ncclInvalidArgument, "%s: null communicator", name);
  else if (dtype < 0 || dtype >= ncclNumTypes)
    rc = fail(ncclInvalidArgument, "rank %d: %s: unknown data type %d", comm->rank, name, dtype);
  else if (kind == KIND_ALLREDUCE && (op != ncclSum || (dtype != ncclUint8 && dtype != ncclUint32 && dtype != ncclUint64 &&
                                                        dtype != ncclFloat64)))
    rc = fail(ncclInvalidArgument, "rank %d: %s: only sums of u8, u32, u64 and f64 are implemented (dtype %d, op %d)", comm->rank,
              name, dtype, op);
  else if (kind == KIND_BROADCAST && (root < 0 || root >= comm->s->nranks))
    rc = fail(ncclInvalidArgument, "rank %d: %s: root %d of %d ranks", comm->rank, name, root, comm->s->nranks);
  else if (count && (!recv || (!send && (kind != KIND_BROADCAST || root == comm->rank))))
    rc = fail(ncclInvalidArgument, "rank %d: %s: null buffer", comm->rank, name);
  else if (t_grp.depth > 0 && t_grp.comm && t_grp.comm != comm)
    rc = fail(ncclInvalidUsage, "rank %d: %s: one group spans two communicators", comm->rank, name);
  if (rc != ncclSuccess) {
    if (t_grp.depth > 0) t_grp.failed = 1;
    return rc;
  }
  if (t_grp.depth == 0) return run_step(comm, &o, 1);
  if (t_grp.n == t_grp.cap) {
    size_t cap = t_grp.cap ? (size_t)t_grp.cap * 2 : 64;
    Op* q = (Op*)realloc(t_grp.ops, cap * sizeof *q);
    if (!q) {
      t_grp.failed = 1;
      return fail(ncclSystemError, "out of host memory");
    }
    t_grp.ops = q;
    t_grp.cap = (int)cap;
  }
  t_grp.comm = comm;
  t_grp.ops[t_grp.n++] = o;
  return ncclSuccess;
}

ncclResult_t ncclBroadcast(const void* send, void* recv, size_t count, int dtype, int root, ncclComm_t comm, void* stream) {
  return enqueue(KIND_BROADCAST, send, recv, count, dtype, ncclSum, root, comm, stream);
}

ncclResult_t ncclAllGather(const void* send, void* recv, size_t count, int dtype, ncclComm_t comm, void* stream) {
  return enqueue(KIND_ALLGATHER, send, recv, count, dtype, ncclSum, -1, comm, stream);
}

ncclResult_t ncclAllReduce(const void* send, void* recv, size_t count, int dtype, int op, ncclComm_t comm, void* stream) {
  return enqueue(KIND_ALLREDUCE, send, recv, count, dtype, op, -1, comm, stream);
}

ncclResult_t ncclGroupStart(void) {
  t_grp.depth++;
  return ncclSuccess;
}

ncclResult_t ncclGroupEnd(void) {
  if (t_grp.depth == 0) return fail(ncclInvalidUsage, "ncclGroupEnd without ncclGroupStart");
  if (--t_grp.depth > 0) return ncclSuccess;
  struct ncclComm* c = t_grp.comm;
  int n = t_grp.n, failed = t_grp.failed;
  t_grp.comm = NULL;
  t_grp.n = 0;
  t_grp.failed = 0;
  if (failed) return ncclInvalidUsage;  // the message of the rejected call stays in t_err
  if (n == 0) return ncclSuccess;
  return run_step(c, t_grp.ops, n);
}
