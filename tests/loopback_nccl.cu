// loopback_nccl.cu — a stand-in for libnccl.so.2 that runs R ranks of ONE process on ONE GPU.
//
// NCCL refuses two ranks on one device, so the multi-rank merge of libalazgpu (alz_comm.cu) could only be
// tested on several GPUs. The library loads NCCL with dlopen("libnccl.so.2") and has no RPATH, so a process
// whose LD_LIBRARY_PATH names the directory of this library gets these six entry points instead:
//   ncclGetUniqueId, ncclCommInitRank, ncclCommDestroy, ncclAllGather, ncclAllReduce (sum), ncclGetErrorString.
//
// A communicator is keyed by the unique-id bytes; ncclCommInitRank is a rendezvous of its ranks (threads).
// A collective is three host barriers of the R calling threads:
//   1. every rank made the same call (op, count, type, reduction) or every rank gets ncclInvalidUsage;
//      each rank records a "ready" event on its stream (an all-reduce first copies its input to staging);
//   2. each stream waits on every peer's ready event, does its copies or its sum kernel, records "done";
//   3. each stream waits on every done event, so no send buffer is reused while a peer still reads it.
// The GPU only ever waits on events that were recorded before the wait was enqueued, so a device-wide
// synchronisation in a rank thread (a cudaFree) cannot deadlock. Every barrier has a host timeout
// (LOOPBACK_NCCL_TIMEOUT_S, default 60 s) after which the communicator is broken and returns ncclSystemError.
//
// Test exports: a per-rank log of (op, bytes) and one fault-free knob that overwrites one rank's
// BlockHeader.status in the k-th block gather, which is what a peer whose local preparation failed sends.
#include <cuda_runtime.h>
#include <nccl.h>

#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

namespace {

constexpr int kOpAllGather = 1, kOpAllReduce = 2;
constexpr size_t kRowWords64 = 37;        // alz_edge_out is 296 bytes
constexpr size_t kMinBlockRows = 1025;    // header row + block_rows_for(0) = 1024 rows

struct Call {
  int op;
  size_t count;
  int type;
  int redop;
  bool operator!=(const Call& o) const { return op != o.op || count != o.count || type != o.type || redop != o.redop; }
};

struct Comm {
  int nranks = 0;
  std::mutex mu;
  std::condition_variable cv;
  int arrived = 0, refs = 0;
  uint64_t gen = 0;
  bool broken = false, mismatch = false;
  bool fault_this = false;              // this round is the block gather the knob names
  std::vector<Call> call;
  std::vector<const void*> send;
  std::vector<void*> recv;
  std::vector<cudaStream_t> stream;
  std::vector<cudaEvent_t> ready, done;
  char* staging = nullptr;              // all-reduce: R input slices
  size_t staging_bytes = 0;
};

}  // namespace

struct ncclComm {
  Comm* c;
  int rank;
};

namespace {

std::mutex g_mu;                          // registry, log, knob
std::map<std::string, Comm*> g_pending;   // communicators whose ranks are still joining
uint64_t g_id_counter = 0;
std::vector<std::vector<std::pair<int, unsigned long long>>> g_log(64);
long g_block_gathers = 0;
int g_fault_rank = -1, g_fault_status = 0;
long g_fault_kth = 0;

double timeout_s() {
  const char* e = getenv("LOOPBACK_NCCL_TIMEOUT_S");
  const double t = e ? atof(e) : 0.0;
  return t > 0.0 ? t : 60.0;
}

// all nranks threads arrive; the last one runs `leader` (under the lock) before anyone leaves
bool barrier(Comm* c, const std::function<void()>& leader) {
  std::unique_lock<std::mutex> lk(c->mu);
  if (c->broken) return false;
  const uint64_t g = c->gen;
  if (++c->arrived == c->nranks) {
    if (leader) leader();
    c->arrived = 0;
    c->gen++;
    c->cv.notify_all();
    return !c->broken;
  }
  const bool ok = c->cv.wait_for(lk, std::chrono::duration<double>(timeout_s()),
                                 [&] { return c->gen != g || c->broken; });
  if (!ok) { c->broken = true; c->cv.notify_all(); }
  return !c->broken;
}

size_t type_bytes(ncclDataType_t t) {
  switch (t) {
    case ncclInt8: case ncclUint8: return 1;
    case ncclFloat16: return 2;
    case ncclInt32: case ncclUint32: case ncclFloat32: return 4;
    case ncclInt64: case ncclUint64: case ncclFloat64: return 8;
    default: return 0;
  }
}

template <typename T>
__global__ void sum_slices_kernel(const T* __restrict__ staging, size_t count, int R, T* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x) {
    T s = 0;
    for (int p = 0; p < R; ++p) s += staging[(size_t)p * count + i];   // integer sums: wrap like NCCL's
    out[i] = s;
  }
}

__global__ void poke_i32_kernel(int32_t* p, int32_t v) { *p = v; }

#define CU(expr) do { if ((expr) != cudaSuccess) return ncclUnhandledCudaError; } while (0)

ncclResult_t collective(ncclComm* me, const Call& call, const void* sendbuff, void* recvbuff, cudaStream_t s) {
  Comm* c = me->c;
  const int r = me->rank, R = c->nranks;
  const size_t tb = type_bytes((ncclDataType_t)call.type);
  if (tb == 0) return ncclInvalidArgument;
  const size_t bytes = call.count * tb;
  {
    std::lock_guard<std::mutex> g(g_mu);
    if (r < (int)g_log.size())
      g_log[r].emplace_back(call.op, (unsigned long long)(call.op == kOpAllGather ? bytes * R : bytes));
  }
  {
    std::lock_guard<std::mutex> g(c->mu);
    c->call[r] = call; c->send[r] = sendbuff; c->recv[r] = recvbuff; c->stream[r] = s;
  }
  bool cuda_ok = true;
  const bool b1 = barrier(c, [&] {
    c->mismatch = false;
    for (int p = 1; p < R; ++p) c->mismatch |= c->call[p] != c->call[0];
    c->fault_this = false;
    if (c->mismatch) return;
    if (call.op == kOpAllGather && call.type == ncclUint64 && call.count % kRowWords64 == 0 &&
        call.count >= kRowWords64 * kMinBlockRows) {
      std::lock_guard<std::mutex> g(g_mu);
      c->fault_this = ++g_block_gathers == g_fault_kth && g_fault_rank >= 0 && g_fault_rank < R;
    }
    if (call.op == kOpAllReduce && bytes * R > c->staging_bytes) {
      cuda_ok = cudaDeviceSynchronize() == cudaSuccess && cudaFree(c->staging) == cudaSuccess;
      c->staging = nullptr;
      c->staging_bytes = 0;
      if (cuda_ok && cudaMalloc(&c->staging, bytes * R) == cudaSuccess) c->staging_bytes = bytes * R;
      else { cuda_ok = false; c->broken = true; }
    }
  });
  if (!b1) return cuda_ok ? ncclSystemError : ncclUnhandledCudaError;
  if (c->mismatch) return ncclInvalidUsage;
  if (call.op == kOpAllReduce && bytes)
    CU(cudaMemcpyAsync(c->staging + (size_t)r * bytes, sendbuff, bytes, cudaMemcpyDeviceToDevice, s));
  CU(cudaEventRecord(c->ready[r], s));
  if (!barrier(c, nullptr)) return ncclSystemError;
  for (int p = 0; p < R; ++p) CU(cudaStreamWaitEvent(s, c->ready[p], 0));
  if (call.op == kOpAllGather) {
    for (int p = 0; p < R; ++p) {
      char* dst = static_cast<char*>(recvbuff) + (size_t)p * bytes;
      if (bytes && dst != c->send[p]) CU(cudaMemcpyAsync(dst, c->send[p], bytes, cudaMemcpyDeviceToDevice, s));
    }
    if (c->fault_this) {
      int status;
      int victim;
      {
        std::lock_guard<std::mutex> g(g_mu);
        status = g_fault_status;
        victim = g_fault_rank;
      }
      int32_t* st = reinterpret_cast<int32_t*>(static_cast<char*>(recvbuff) + (size_t)victim * bytes + 8);
      poke_i32_kernel<<<1, 1, 0, s>>>(st, status);
      CU(cudaGetLastError());
    }
  } else if (call.count) {
    const unsigned grid = (unsigned)std::min<size_t>((call.count + 255) / 256, 1024);
    if (tb == 8) sum_slices_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const uint64_t*>(c->staging), call.count, R,
                                                        static_cast<uint64_t*>(recvbuff));
    else sum_slices_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const uint32_t*>(c->staging), call.count, R,
                                                static_cast<uint32_t*>(recvbuff));
    CU(cudaGetLastError());
  }
  CU(cudaEventRecord(c->done[r], s));
  if (!barrier(c, nullptr)) return ncclSystemError;
  for (int p = 0; p < R; ++p) CU(cudaStreamWaitEvent(s, c->done[p], 0));
  return ncclSuccess;
}

}  // namespace

extern "C" {

ncclResult_t ncclGetUniqueId(ncclUniqueId* id) {
  if (!id) return ncclInvalidArgument;
  memset(id, 0, sizeof(*id));
  std::lock_guard<std::mutex> g(g_mu);
  const uint64_t words[3] = {0x6C6F6F706261636Bull, (uint64_t)getpid(), ++g_id_counter};
  memcpy(id->internal, words, sizeof(words));
  return ncclSuccess;
}

ncclResult_t ncclCommInitRank(ncclComm_t* out, int nranks, ncclUniqueId id, int rank) {
  if (!out || nranks < 1 || rank < 0 || rank >= nranks) return ncclInvalidArgument;
  const std::string key(id.internal, sizeof(id.internal));
  Comm* c;
  {
    std::lock_guard<std::mutex> g(g_mu);
    auto it = g_pending.find(key);
    if (it == g_pending.end()) {
      c = new Comm();
      c->nranks = nranks;
      c->call.resize(nranks); c->send.resize(nranks); c->recv.resize(nranks); c->stream.resize(nranks);
      c->ready.resize(nranks); c->done.resize(nranks);
      for (int p = 0; p < nranks; ++p) {
        if (cudaEventCreateWithFlags(&c->ready[p], cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&c->done[p], cudaEventDisableTiming) != cudaSuccess)
          return ncclUnhandledCudaError;
      }
      g_pending[key] = c;
    } else {
      c = it->second;
    }
    if (c->nranks != nranks) return ncclInvalidUsage;
    c->refs++;
  }
  // the rendezvous: once every rank has joined, the id is free for a new communicator
  if (!barrier(c, [&] {
        std::lock_guard<std::mutex> g(g_mu);
        g_pending.erase(key);
      }))
    return ncclSystemError;
  *out = new ncclComm{c, rank};
  return ncclSuccess;
}

ncclResult_t ncclCommDestroy(ncclComm_t comm) {
  if (!comm) return ncclInvalidArgument;
  Comm* c = comm->c;
  delete comm;
  bool last;
  {
    std::lock_guard<std::mutex> g(g_mu);
    last = --c->refs == 0;
  }
  if (last) {
    cudaDeviceSynchronize();
    for (int p = 0; p < c->nranks; ++p) { cudaEventDestroy(c->ready[p]); cudaEventDestroy(c->done[p]); }
    cudaFree(c->staging);
    delete c;
  }
  return ncclSuccess;
}

ncclResult_t ncclAllGather(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t type, ncclComm_t comm,
                           cudaStream_t stream) {
  if (!comm) return ncclInvalidArgument;
  return collective(comm, Call{kOpAllGather, count, (int)type, -1}, sendbuff, recvbuff, stream);
}

ncclResult_t ncclAllReduce(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t type, ncclRedOp_t op,
                           ncclComm_t comm, cudaStream_t stream) {
  if (!comm) return ncclInvalidArgument;
  if (op != ncclSum || (type_bytes(type) != 4 && type_bytes(type) != 8) || type == ncclFloat32 || type == ncclFloat64)
    return ncclInvalidArgument;   // the sums the merge uses: integers
  return collective(comm, Call{kOpAllReduce, count, (int)type, (int)op}, sendbuff, recvbuff, stream);
}

const char* ncclGetErrorString(ncclResult_t r) {
  switch (r) {
    case ncclSuccess: return "no error";
    case ncclUnhandledCudaError: return "loopback: CUDA call failed";
    case ncclSystemError: return "loopback: barrier timed out or communicator broken";
    case ncclInvalidArgument: return "loopback: invalid argument";
    case ncclInvalidUsage: return "loopback: ranks disagree on the collective";
    default: return "loopback: error";
  }
}

// ---- test exports ----
// log of rank r: n entries of (op: 1 all-gather, 2 all-reduce; bytes: all-gather received, all-reduce reduced)
int loopback_log_count(int rank) {
  std::lock_guard<std::mutex> g(g_mu);
  return rank >= 0 && rank < (int)g_log.size() ? (int)g_log[rank].size() : -1;
}
int loopback_log_entry(int rank, int i, int* op, unsigned long long* bytes) {
  std::lock_guard<std::mutex> g(g_mu);
  if (rank < 0 || rank >= (int)g_log.size() || i < 0 || i >= (int)g_log[rank].size()) return -1;
  *op = g_log[rank][i].first;
  *bytes = g_log[rank][i].second;
  return 0;
}
void loopback_log_clear(void) {
  std::lock_guard<std::mutex> g(g_mu);
  for (auto& l : g_log) l.clear();
}
// the kth (1-based, counted from now) block gather delivers `status` as rank `rank`'s BlockHeader.status to
// every rank; rank < 0 disarms
void loopback_fault_block_status(int rank, long kth, int status) {
  std::lock_guard<std::mutex> g(g_mu);
  g_block_gathers = 0;
  g_fault_rank = rank;
  g_fault_kth = kth;
  g_fault_status = status;
}

}  // extern "C"
