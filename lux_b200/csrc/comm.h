// comm.h — NCCL bound at run time with dlopen, so that libluxb.so loads (and all single-GPU paths work) on hosts
// without NCCL and never clashes with the copy torch bundles.  Replaces the implicit exchange the reference gets
// from Legion regions in zero-copy memory (SURVEY §2.1): (a) all-gather of vertex-value slices, (b) all-gather of
// frontier slots, (c) sum of per-partition active counts / out-degree histograms.
#pragma once
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stddef.h>
#include <stdint.h>
#include <mutex>

namespace luxb {

typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef enum { ncclSuccess = 0 } ncclResult_t;
// values from nccl.h (stable across NCCL 2.x)
enum { ncclInt8 = 0, ncclUint8 = 1, ncclInt32 = 2, ncclUint32 = 3, ncclInt64 = 4, ncclUint64 = 5, ncclFloat32 = 7, ncclFloat64 = 8 };
enum { ncclSum = 0 };

struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;

  // returns nullptr on success, else a message.  Thread-safe: one host thread per GPU may race here.
  const char* load() {
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    if (handle && GetErrorString) return nullptr;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (handle) break;
    }
    if (!handle) return "cannot dlopen libnccl.so.2";
#define LUXB_SYM(field, name)                                   \
  field = reinterpret_cast<decltype(field)>(dlsym(handle, name)); \
  if (!field) return "missing NCCL symbol " name;
    LUXB_SYM(GetUniqueId, "ncclGetUniqueId")
    LUXB_SYM(CommInitRank, "ncclCommInitRank")
    LUXB_SYM(CommDestroy, "ncclCommDestroy")
    LUXB_SYM(AllReduce, "ncclAllReduce")
    LUXB_SYM(Broadcast, "ncclBroadcast")
    LUXB_SYM(AllGather, "ncclAllGather")
    LUXB_SYM(GroupStart, "ncclGroupStart")
    LUXB_SYM(GroupEnd, "ncclGroupEnd")
    LUXB_SYM(GetErrorString, "ncclGetErrorString")
#undef LUXB_SYM
    return nullptr;
  }
};

inline NcclApi& nccl() {
  static NcclApi api;
  return api;
}

}  // namespace luxb
