// An in-process NCCL stand-in for tests: the eight entry points libb2kmeans resolves (csrc/b2k_comm.cu), for ranks
// that live as threads of one process and may share one GPU, which real NCCL refuses.  Loaded through B2K_NCCL_LIB.
//
// Every collective is host-synchronous: the caller's stream is synchronised, its buffer copied to the host, the ranks
// meet at the group's next rendezvous, the last rank to arrive forms the result once, and every rank copies it back.
// Nothing ever waits on the GPU for another rank, so a missing rank shows up as a host-side timeout, not a hang.
//
//   AllReduce(sum)  summed once, in rank order, in the dtype's own arithmetic: every rank receives identical bits, as
//                   NCCL guarantees (NCCL's own order differs; this one is rank 0 + rank 1 + ... left to right).
//   AllGather       rank-order concatenation of snapshots of `send` taken before the rendezvous, so `send` may alias
//                   the caller's own slot of `recv`.
//   sequence check  every rank must present the same (op, dtype, count) at a rendezvous; otherwise every rank fails
//                   with a message naming the rendezvous number and each rank's call.  Real NCCL would hang there.
//   timeout         a rendezvous (or CommInitRank) still missing a rank after B2K_FAKE_NCCL_TIMEOUT_S seconds
//                   (default 30) fails on every waiting rank, naming the missing ranks.
//   abort           CommAbort wakes every waiter with an error.
// After any failure the group is broken: every later call on it fails with the same message.  GetErrorString(rc)
// returns the code's name followed by the calling thread's last failure message, which is where the detail reaches
// b2k_last_error.
//
// Two extra entry points serve the tests: b2kFakeNcclTrace (the collectives one rank of a group issued) and
// b2kFakeNcclGroupError (the message that broke a group).
#include <cuda_runtime.h>

#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

namespace {

// NCCL's ABI: ncclResult_t, ncclDataType_t and ncclRedOp_t values
enum { kSuccess = 0, kUnhandledCudaError = 1, kSystemError = 2, kInternalError = 3, kInvalidArgument = 4,
       kInvalidUsage = 5, kRemoteError = 6 };
enum { kInt8 = 0, kUint8 = 1, kInt32 = 2, kUint32 = 3, kInt64 = 4, kUint64 = 5, kFloat16 = 6, kFloat32 = 7,
       kFloat64 = 8 };
enum { kSum = 0 };
enum { kOpAllReduce = 0, kOpAllGather = 1 };

struct UniqueId { char internal[128]; };

const char* op_name(int op) { return op == kOpAllReduce ? "AllReduce" : "AllGather"; }

size_t dtype_size(int dt) {
  switch (dt) {
    case kUint8: return 1;
    case kInt64: return 8;
    case kFloat32: return 4;
    case kFloat64: return 8;
    default: return 0;   // not used by libb2kmeans: rejected
  }
}

double timeout_s() {
  const char* e = std::getenv("B2K_FAKE_NCCL_TIMEOUT_S");
  double t = e ? std::atof(e) : 30.0;
  return t > 0 ? t : 30.0;
}

thread_local std::string t_last_msg;   // detail of this thread's last failure (GetErrorString)

int fail(int rc, const std::string& msg) {
  t_last_msg = msg;
  return rc;
}

struct Call {   // one rank's part of one rendezvous
  int op = 0, dtype = 0;
  size_t count = 0;
  std::vector<char> data;
};

struct Group {
  std::mutex m;
  std::condition_variable cv;
  int nranks = 0;
  std::vector<int> joined;               // CommInitRank seen per rank
  int n_joined = 0;
  std::string error;                     // non-empty: the group is broken
  // the rendezvous being gathered: number `gen`; ranks fill `calls`, the last one forms `result`
  uint64_t gen = 0;
  std::vector<int> present;
  int arrived = 0, departed = 0;
  bool ready = false;
  std::vector<Call> calls;
  std::vector<char> result;
  std::vector<std::vector<std::string>> trace;   // per rank: "op dtype count" of every collective it entered

  void break_group(const std::string& msg) {   // m held
    if (error.empty()) error = msg;
    cv.notify_all();
  }
  std::string missing() const {   // m held
    std::string s;
    for (int r = 0; r < nranks; ++r)
      if (!present[r]) s += (s.empty() ? "" : ", ") + std::to_string(r);
    return s;
  }
};

std::mutex g_reg_m;
std::map<std::string, std::shared_ptr<Group>> g_groups;   // kept after destroy: the tests read traces afterwards
uint64_t g_next_id = 0;

std::shared_ptr<Group> find_group(const UniqueId& id) {
  std::lock_guard<std::mutex> lk(g_reg_m);
  auto it = g_groups.find(std::string(id.internal, sizeof(id.internal)));
  return it == g_groups.end() ? nullptr : it->second;
}

}  // namespace

struct ncclComm {
  std::shared_ptr<Group> g;
  int rank = 0;
  uint64_t seq = 0;   // collectives this rank entered
};

namespace {

std::string describe(const Call& c) {
  return std::string(op_name(c.op)) + "(dtype " + std::to_string(c.dtype) + ", count " + std::to_string(c.count) + ")";
}

template <typename T>
void sum_into(std::vector<char>& acc, const std::vector<char>& add, size_t count) {
  T* a = reinterpret_cast<T*>(acc.data());
  const T* b = reinterpret_cast<const T*>(add.data());
  for (size_t i = 0; i < count; ++i) a[i] = (T)(a[i] + b[i]);
}

void form_result(Group& g) {   // m held; every call matched
  const Call& c0 = g.calls[0];
  const size_t bytes = c0.count * dtype_size(c0.dtype);
  if (c0.op == kOpAllGather) {
    g.result.resize(bytes * g.nranks);
    for (int r = 0; r < g.nranks; ++r)
      if (bytes) std::memcpy(g.result.data() + r * bytes, g.calls[r].data.data(), bytes);
    return;
  }
  g.result = g.calls[0].data;
  for (int r = 1; r < g.nranks; ++r) {
    switch (c0.dtype) {
      case kUint8: sum_into<uint8_t>(g.result, g.calls[r].data, c0.count); break;
      case kInt64: sum_into<int64_t>(g.result, g.calls[r].data, c0.count); break;
      case kFloat32: sum_into<float>(g.result, g.calls[r].data, c0.count); break;
      case kFloat64: sum_into<double>(g.result, g.calls[r].data, c0.count); break;
    }
  }
}

// Enters this rank's next rendezvous with `call`; on success `out` holds the result.
int rendezvous(ncclComm* comm, Call&& call, std::vector<char>* out) {
  Group& g = *comm->g;
  const uint64_t my = comm->seq++;
  const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(timeout_s());
  std::unique_lock<std::mutex> lk(g.m);
  g.trace[comm->rank].push_back(std::to_string(call.op) + " " + std::to_string(call.dtype) + " " +
                                std::to_string(call.count));
  auto timed_out = [&](const char* what) {
    g.break_group("fake NCCL: rendezvous #" + std::to_string(my) + " (" + describe(call) + " from rank " +
                  std::to_string(comm->rank) + ") timed out after " + std::to_string((int)timeout_s()) + " s " + what +
                  "; missing ranks: " + g.missing());
  };
  // the previous rendezvous must be fully consumed before this one gathers
  while (g.error.empty() && g.gen != my) {
    if (g.gen > my) {
      g.break_group("fake NCCL: rank " + std::to_string(comm->rank) + " entered rendezvous #" + std::to_string(my) +
                    " after the group moved past it");
      break;
    }
    if (g.cv.wait_until(lk, deadline) == std::cv_status::timeout && g.gen != my) timed_out("waiting to start");
  }
  if (!g.error.empty()) return fail(kRemoteError, g.error);
  g.calls[comm->rank] = std::move(call);
  g.present[comm->rank] = 1;
  if (++g.arrived == g.nranks) {
    bool same = true;
    for (int r = 1; r < g.nranks; ++r) {
      const Call &a = g.calls[0], &b = g.calls[r];
      same = same && a.op == b.op && a.dtype == b.dtype && a.count == b.count;
    }
    if (!same) {
      std::string m = "fake NCCL: collective sequence mismatch at rendezvous #" + std::to_string(my) + ":";
      for (int r = 0; r < g.nranks; ++r) m += " rank " + std::to_string(r) + " " + describe(g.calls[r]) + ";";
      g.break_group(m);
      return fail(kInvalidUsage, g.error);
    }
    form_result(g);
    g.ready = true;
    g.cv.notify_all();
  }
  while (g.error.empty() && !g.ready)
    if (g.cv.wait_until(lk, deadline) == std::cv_status::timeout && !g.ready) timed_out("waiting for its peers");
  if (!g.error.empty()) return fail(kRemoteError, g.error);
  *out = g.result;
  if (++g.departed == g.nranks) {   // the last one out opens the next rendezvous
    g.arrived = g.departed = 0;
    g.ready = false;
    for (auto& p : g.present) p = 0;
    for (auto& c : g.calls) c = Call{};
    g.result.clear();
    ++g.gen;
    g.cv.notify_all();
  }
  return kSuccess;
}

int check_comm(ncclComm* comm) {
  if (!comm || !comm->g) return fail(kInvalidArgument, "fake NCCL: NULL communicator");
  return kSuccess;
}

int to_host(const void* dev, size_t bytes, std::vector<char>* out, cudaStream_t s) {
  out->resize(bytes);
  cudaError_t e = cudaStreamSynchronize(s);
  if (e == cudaSuccess && bytes) e = cudaMemcpyAsync(out->data(), dev, bytes, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return fail(kUnhandledCudaError, std::string("fake NCCL: ") + cudaGetErrorString(e));
  return kSuccess;
}

int to_device(void* dev, const std::vector<char>& in, cudaStream_t s) {
  cudaError_t e = in.empty() ? cudaSuccess : cudaMemcpyAsync(dev, in.data(), in.size(), cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);   // `in` is pageable and dies with the caller's frame
  if (e != cudaSuccess) return fail(kUnhandledCudaError, std::string("fake NCCL: ") + cudaGetErrorString(e));
  return kSuccess;
}

}  // namespace

extern "C" {

int ncclGetVersion(int* version) {
  if (!version) return fail(kInvalidArgument, "fake NCCL: version is NULL");
  *version = 22105;   // reports itself as NCCL 2.21.5
  return kSuccess;
}

int ncclGetUniqueId(UniqueId* id) {
  if (!id) return fail(kInvalidArgument, "fake NCCL: id is NULL");
  std::memset(id->internal, 0, sizeof(id->internal));
  uint64_t n;
  {
    std::lock_guard<std::mutex> lk(g_reg_m);
    n = ++g_next_id;
  }
  std::snprintf(id->internal, sizeof(id->internal), "b2k-fake-nccl:%llu", (unsigned long long)n);
  return kSuccess;
}

int ncclCommInitRank(ncclComm** comm, int nranks, UniqueId id, int rank) {
  if (!comm || nranks < 1 || rank < 0 || rank >= nranks)
    return fail(kInvalidArgument, "fake NCCL: bad comm/nranks/rank");
  std::shared_ptr<Group> gp;
  {
    std::lock_guard<std::mutex> lk(g_reg_m);
    auto& slot = g_groups[std::string(id.internal, sizeof(id.internal))];
    if (!slot) {
      slot = std::make_shared<Group>();
      slot->nranks = nranks;
      slot->joined.assign(nranks, 0);
      slot->present.assign(nranks, 0);
      slot->calls.resize(nranks);
      slot->trace.resize(nranks);
    }
    gp = slot;
  }
  Group& g = *gp;
  std::unique_lock<std::mutex> lk(g.m);
  if (g.nranks != nranks)
    return fail(kInvalidUsage, "fake NCCL: rank " + std::to_string(rank) + " joins with nranks " +
                                   std::to_string(nranks) + ", the group has " + std::to_string(g.nranks));
  if (g.joined[rank]) return fail(kInvalidUsage, "fake NCCL: duplicate rank " + std::to_string(rank));
  g.joined[rank] = 1;
  if (++g.n_joined == g.nranks) g.cv.notify_all();
  const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(timeout_s());
  while (g.error.empty() && g.n_joined < g.nranks) {
    if (g.cv.wait_until(lk, deadline) == std::cv_status::timeout && g.n_joined < g.nranks) {
      std::string miss;
      for (int r = 0; r < g.nranks; ++r)
        if (!g.joined[r]) miss += (miss.empty() ? "" : ", ") + std::to_string(r);
      g.break_group("fake NCCL: CommInitRank timed out after " + std::to_string((int)timeout_s()) +
                    " s; missing ranks: " + miss);
    }
  }
  if (!g.error.empty()) return fail(kRemoteError, g.error);
  *comm = new ncclComm{gp, rank, 0};
  return kSuccess;
}

int ncclCommDestroy(ncclComm* comm) {
  if (int rc = check_comm(comm)) return rc;
  delete comm;
  return kSuccess;
}

int ncclCommAbort(ncclComm* comm) {
  if (int rc = check_comm(comm)) return rc;
  {
    std::lock_guard<std::mutex> lk(comm->g->m);
    comm->g->break_group("fake NCCL: communicator aborted by rank " + std::to_string(comm->rank));
  }
  delete comm;
  return kSuccess;
}

int ncclAllReduce(const void* send, void* recv, size_t count, int dtype, int op, ncclComm* comm, cudaStream_t s) {
  if (int rc = check_comm(comm)) return rc;
  if (!dtype_size(dtype) || op != kSum)
    return fail(kInvalidArgument, "fake NCCL: AllReduce supports sum of uint8, int64, float32 and float64 only");
  Call c;
  c.op = kOpAllReduce;
  c.dtype = dtype;
  c.count = count;
  if (int rc = to_host(send, count * dtype_size(dtype), &c.data, s)) return rc;
  std::vector<char> res;
  if (int rc = rendezvous(comm, std::move(c), &res)) return rc;
  return to_device(recv, res, s);
}

int ncclAllGather(const void* send, void* recv, size_t sendcount, int dtype, ncclComm* comm, cudaStream_t s) {
  if (int rc = check_comm(comm)) return rc;
  if (!dtype_size(dtype)) return fail(kInvalidArgument, "fake NCCL: AllGather of an unsupported dtype");
  Call c;
  c.op = kOpAllGather;
  c.dtype = dtype;
  c.count = sendcount;
  if (int rc = to_host(send, sendcount * dtype_size(dtype), &c.data, s)) return rc;
  std::vector<char> res;
  if (int rc = rendezvous(comm, std::move(c), &res)) return rc;
  return to_device(recv, res, s);
}

const char* ncclGetErrorString(int rc) {
  static const char* names[] = {"no error", "unhandled cuda error", "unhandled system error", "internal error",
                                "invalid argument", "invalid usage", "remote process exited or there was a network error"};
  const char* base = rc >= 0 && rc <= kRemoteError ? names[rc] : "unknown result code";
  thread_local std::string s;
  s = base;
  if (rc != kSuccess && !t_last_msg.empty()) s += ": " + t_last_msg;
  return s.c_str();
}

// The collectives `rank` of the group keyed by `id` entered, one "op dtype count" line each (op 0 = AllReduce,
// 1 = AllGather).  Returns the length written without the terminator, -1 for an unknown group or rank, or the
// length needed when `cap` is too small.
long long b2kFakeNcclTrace(const UniqueId* id, int rank, char* buf, long long cap) {
  std::shared_ptr<Group> g = id ? find_group(*id) : nullptr;
  if (!g) return -1;
  std::lock_guard<std::mutex> lk(g->m);
  if (rank < 0 || rank >= g->nranks) return -1;
  std::string s;
  for (const auto& l : g->trace[rank]) s += l + "\n";
  if ((long long)s.size() + 1 > cap) return (long long)s.size() + 1;
  std::memcpy(buf, s.c_str(), s.size() + 1);
  return (long long)s.size();
}

// The message that broke the group keyed by `id` ("" while it is healthy); same return rules as b2kFakeNcclTrace.
long long b2kFakeNcclGroupError(const UniqueId* id, char* buf, long long cap) {
  std::shared_ptr<Group> g = id ? find_group(*id) : nullptr;
  if (!g) return -1;
  std::lock_guard<std::mutex> lk(g->m);
  if ((long long)g->error.size() + 1 > cap) return (long long)g->error.size() + 1;
  std::memcpy(buf, g->error.c_str(), g->error.size() + 1);
  return (long long)g->error.size();
}

}  // extern "C"
