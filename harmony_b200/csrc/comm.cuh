// comm.cuh — NCCL through dlopen (the process usually already holds torch's libnccl.so.2), the process-wide
// communicators and the all-reduces of sharded cells.
#pragma once

namespace {

struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
} g_nccl;

bool load_nccl(std::string* why) {
  if (g_nccl.ok) return true;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* nm : names) {
    g_nccl.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
    if (g_nccl.lib) break;
  }
  if (!g_nccl.lib) {
    if (why) *why = "cannot dlopen libnccl.so.2";
    return false;
  }
#define L(sym) *(void**)(&g_nccl.sym) = dlsym(g_nccl.lib, "nccl" #sym)
  L(GetUniqueId);
  L(CommInitRank);
  L(AllReduce);
  L(AllGather);
  L(CommDestroy);
  L(GetErrorString);
#undef L
  g_nccl.ok = g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.AllReduce && g_nccl.AllGather && g_nccl.CommDestroy;
  if (!g_nccl.ok && why) *why = "libnccl lacks required symbols";
  return g_nccl.ok;
}

#define CKN(call)                                                                                  \
  do {                                                                                             \
    ncclResult_t r__ = (call);                                                                     \
    if (r__ != ncclSuccess)                                                                        \
      return fail(h, 11, "NCCL error %s at %s:%d", g_nccl.GetErrorString ? g_nccl.GetErrorString(r__) : "?", __FILE__, __LINE__); \
  } while (0)

// one NCCL communicator per (device, rank, world) is kept for the life of the process and shared by every
// handle that asks for it with a NULL id (communicator set-up costs ~1 s; models come and go)
struct CommKey {
  int device, rank, world;
  bool operator<(const CommKey& o) const {
    return std::tie(device, rank, world) < std::tie(o.device, o.rank, o.world);
  }
};
std::map<CommKey, ncclComm_t> g_comms;

int allreduce_f(hb_handle* h, float* p, size_t count) {
  if (h->world <= 1) return 0;
  CKN(g_nccl.AllReduce(p, p, count, ncclFloat, ncclSum, h->comm, h->stream));
  return 0;
}
int allreduce_d(hb_handle* h, double* p, size_t count) {
  if (h->world <= 1) return 0;
  CKN(g_nccl.AllReduce(p, p, count, ncclDouble, ncclSum, h->comm, h->stream));
  return 0;
}

}  // namespace
