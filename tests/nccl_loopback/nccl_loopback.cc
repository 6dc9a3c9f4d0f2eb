// nccl_loopback.cc — an NCCL stand-in whose ranks are threads of one process on one GPU.
//
// The sharded index (dingo-store_b200/csrc/shard.cu) resolves NCCL at run time and tries B200VS_NCCL_LIB first.  Real NCCL
// refuses two ranks on one device, so a test that wants worlds of 2..8 on a single GPU points B200VS_NCCL_LIB at this
// library and runs each rank in a thread (tests/shard_loopback.py).  It implements only the entry points shard.cu uses.
//
// Every collective call meets its peers in a host rendezvous keyed by the communicator's call counter; the ranks must agree
// on the operation, count, datatype and root, or every rank returns ncclInvalidUsage and the mismatch is printed on stderr
// (a desynchronised product is exactly what the tests look for).  Every host wait is timed and returns ncclSystemError on
// expiry, so a bug fails a test instead of hanging it; no device work ever waits for work that has not been enqueued.
//
// AllGather, Broadcast and Send / Recv are stream-ordered, not host-synchronised: each rank records an event on its stream
// when it posts, the readers' streams wait on it before their copies, and after a second rendezvous each writer's stream
// waits on its readers' "read done" events, so no buffer is reused before it has been read.  AllReduce stages through the
// host.  Streams are driven through the driver API: the caller's runtime may be linked statically, and the driver is the
// one object both sides share.
#include <cuda.h>
#include <nccl.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

namespace {

constexpr auto kTimeout = std::chrono::seconds(60);

enum Op { OP_ALLGATHER = 1, OP_BROADCAST, OP_ALLREDUCE, OP_SPLIT };
const char* op_name(int op) {
  switch (op) {
    case OP_ALLGATHER: return "AllGather";
    case OP_BROADCAST: return "Broadcast";
    case OP_ALLREDUCE: return "AllReduce";
    case OP_SPLIT: return "CommSplit";
  }
  return "?";
}

size_t type_size(ncclDataType_t t) {
  switch (t) {
    case ncclInt8: case ncclUint8: return 1;
    case ncclFloat16: case ncclBfloat16: return 2;
    case ncclInt32: case ncclUint32: case ncclFloat32: return 4;
    case ncclInt64: case ncclUint64: case ncclFloat64: return 8;
    default: return 0;
  }
}

// What one rank brings to a collective.
struct Post {
  int op = 0, root = -1, color = 0, key = 0;
  size_t count = 0;
  int dtype = -1;
  const void* send = nullptr;
  void* recv = nullptr;
  CUevent posted = nullptr;     // recorded on the rank's stream when it posted
  CUevent read = nullptr;       // recorded on the rank's stream after its copies
  const void* host = nullptr;   // AllReduce: the rank's values on the host
};

struct Round {
  std::vector<Post> posts;
  int arrived = 0, arrived2 = 0, left = 0;
};

// One point-to-point send waiting in a (src, dst) FIFO.
struct Pending {
  const void* ptr = nullptr;
  size_t bytes = 0;
  CUevent posted = nullptr;
  CUevent read = nullptr;
  bool consumed = false;
  bool bad = false;
};

struct Group {
  std::string key;
  int world = 0;
  int joined = 0, alive = 0;
  std::mutex mu;
  std::condition_variable cv;
  std::map<uint64_t, Round> rounds;
  std::map<std::pair<int, int>, std::deque<std::shared_ptr<Pending>>> fifo;
};

struct Comm {
  Group* g = nullptr;
  int rank = 0, world = 0;
  uint64_t calls = 0;
  std::mutex mu;  // one call at a time per communicator
};

std::mutex g_reg_mu;
std::map<std::string, Group*> g_reg;
std::atomic<uint64_t> g_next_id{1};

void say(const char* fmt, const std::string& a, const std::string& b = "") {
  fprintf(stderr, "[nccl_loopback] ");
  fprintf(stderr, fmt, a.c_str(), b.c_str());
  fprintf(stderr, "\n");
  fflush(stderr);
}

bool cu_ok(CUresult r, const char* what) {
  if (r == CUDA_SUCCESS) return true;
  const char* s = nullptr;
  cuGetErrorString(r, &s);
  fprintf(stderr, "[nccl_loopback] %s failed: %s\n", what, s ? s : "?");
  return false;
}
#define CU(expr) \
  do { if (!cu_ok((expr), #expr)) return ncclUnhandledCudaError; } while (0)

// The driver calls need a current context; the ranks share device 0's primary context (the one the CUDA runtime uses).
bool ensure_ctx() {
  static std::once_flag once;
  static CUcontext primary = nullptr;
  std::call_once(once, [] {
    if (!cu_ok(cuInit(0), "cuInit")) return;
    CUdevice dev;
    if (cu_ok(cuDeviceGet(&dev, 0), "cuDeviceGet")) cu_ok(cuDevicePrimaryCtxRetain(&primary, dev), "cuDevicePrimaryCtxRetain");
  });
  CUcontext cur = nullptr;
  if (cuCtxGetCurrent(&cur) == CUDA_SUCCESS && cur) return true;
  return primary && cu_ok(cuCtxSetCurrent(primary), "cuCtxSetCurrent");
}

std::string desc(const Post& p) {
  return std::string(op_name(p.op)) + "(count " + std::to_string(p.count) + ", datatype " + std::to_string(p.dtype) + ", root " +
         std::to_string(p.root) + ")";
}

// Timed wait on the group's condition variable; false on expiry.
template <class Pred>
bool wait(Group* g, std::unique_lock<std::mutex>& lk, Pred pred, const char* what) {
  if (g->cv.wait_for(lk, kTimeout, pred)) return true;
  fprintf(stderr, "[nccl_loopback] timed out after %lld s waiting for %s (communicator of %d ranks)\n",
          (long long)kTimeout.count(), what, g->world);
  fflush(stderr);
  return false;
}

// First rendezvous of call `seq`: post this rank's part, wait for every peer's, check that they agree.  On success
// `posts` holds every rank's post.  Every rank leaves through leave().
ncclResult_t meet(Comm* c, uint64_t seq, const Post& mine, std::vector<Post>& posts) {
  Group* g = c->g;
  std::unique_lock<std::mutex> lk(g->mu);
  Round& r = g->rounds[seq];
  if (r.posts.empty()) r.posts.resize(g->world);
  r.posts[c->rank] = mine;
  ++r.arrived;
  g->cv.notify_all();
  if (!wait(g, lk, [&] { return r.arrived == g->world; }, op_name(mine.op))) return ncclSystemError;
  posts = r.posts;
  for (int w = 0; w < g->world; ++w) {
    const Post& p = posts[w];
    if (p.op != mine.op || p.count != mine.count || p.dtype != mine.dtype || p.root != mine.root) {
      if (c->rank == 0) say("collective mismatch: %s on one rank, %s on another", desc(mine), desc(p));
      return ncclInvalidUsage;
    }
  }
  return ncclSuccess;
}

// Second rendezvous: publish this rank's "read done" event and wait for every peer's.
ncclResult_t meet2(Comm* c, uint64_t seq, CUevent read, std::vector<Post>& posts) {
  Group* g = c->g;
  std::unique_lock<std::mutex> lk(g->mu);
  Round& r = g->rounds[seq];
  r.posts[c->rank].read = read;
  ++r.arrived2;
  g->cv.notify_all();
  if (!wait(g, lk, [&] { return r.arrived2 == g->world; }, "the second rendezvous")) return ncclSystemError;
  posts = r.posts;
  return ncclSuccess;
}

// The last rank out of call `seq` destroys its events (a stream wait already enqueued on an event survives its destruction).
void leave(Comm* c, uint64_t seq) {
  Group* g = c->g;
  std::lock_guard<std::mutex> lk(g->mu);
  auto it = g->rounds.find(seq);
  if (it == g->rounds.end()) return;
  if (++it->second.left < g->world) return;
  for (Post& p : it->second.posts) {
    if (p.posted) cuEventDestroy(p.posted);
    if (p.read) cuEventDestroy(p.read);
  }
  g->rounds.erase(it);
}

ncclResult_t record(CUevent* e, cudaStream_t s) {
  CU(cuEventCreate(e, CU_EVENT_DISABLE_TIMING));
  CU(cuEventRecord(*e, (CUstream)s));
  return ncclSuccess;
}

Comm* as_comm(ncclComm_t c) { return reinterpret_cast<Comm*>(c); }

ncclResult_t init_rank(Comm** out, int nranks, const std::string& key, int rank) {
  if (!out || nranks < 1 || rank < 0 || rank >= nranks) return ncclInvalidArgument;
  Group* g;
  {
    std::lock_guard<std::mutex> lk(g_reg_mu);
    auto it = g_reg.find(key);
    if (it == g_reg.end()) {
      g = new Group();
      g->key = key;
      g->world = nranks;
      g_reg[key] = g;
    } else {
      g = it->second;
    }
  }
  std::unique_lock<std::mutex> lk(g->mu);
  if (g->world != nranks) {
    say("CommInitRank: world %s disagrees with a peer's %s", std::to_string(nranks), std::to_string(g->world));
    return ncclInvalidUsage;
  }
  ++g->joined;
  ++g->alive;
  g->cv.notify_all();
  if (!wait(g, lk, [&] { return g->joined >= g->world; }, "CommInitRank")) { --g->alive; return ncclSystemError; }
  Comm* c = new Comm();
  c->g = g; c->rank = rank; c->world = nranks;
  *out = c;
  return ncclSuccess;
}

struct P2P {
  bool send;
  Comm* comm;
  int peer;
  void* ptr;
  size_t bytes;
  cudaStream_t stream;
};
thread_local int t_depth = 0;
thread_local std::vector<P2P> t_ops;

ncclResult_t run_group(std::vector<P2P> ops) {
  if (ops.empty()) return ncclSuccess;
  if (!ensure_ctx()) return ncclUnhandledCudaError;
  ncclResult_t rc = ncclSuccess;
  // 1) post every send to its (src, dst) FIFO
  std::vector<std::pair<Group*, std::shared_ptr<Pending>>> sent;
  for (const P2P& o : ops) {
    if (!o.send) continue;
    auto p = std::make_shared<Pending>();
    p->ptr = o.ptr; p->bytes = o.bytes;
    if ((rc = record(&p->posted, o.stream)) != ncclSuccess) return rc;
    Group* g = o.comm->g;
    std::lock_guard<std::mutex> lk(g->mu);
    g->fifo[{o.comm->rank, o.peer}].push_back(p);
    sent.emplace_back(g, p);
    g->cv.notify_all();
  }
  // 2) take every receive from its peer's FIFO, in posting order
  for (const P2P& o : ops) {
    if (o.send) continue;
    Group* g = o.comm->g;
    std::shared_ptr<Pending> p;
    {
      std::unique_lock<std::mutex> lk(g->mu);
      auto& q = g->fifo[{o.peer, o.comm->rank}];
      if (!wait(g, lk, [&] { return !q.empty(); }, "a send matching a Recv")) return ncclSystemError;
      p = q.front();
      q.pop_front();
    }
    bool bad = p->bytes != o.bytes;
    if (bad) {
      say("Send / Recv mismatch: %s bytes sent, %s bytes expected",
          std::to_string(p->bytes), std::to_string(o.bytes) + " (rank " + std::to_string(o.comm->rank) + " from " + std::to_string(o.peer) + ")");
    } else {
      CU(cuStreamWaitEvent((CUstream)o.stream, p->posted, 0));
      if (o.bytes) CU(cuMemcpyAsync((CUdeviceptr)o.ptr, (CUdeviceptr)p->ptr, o.bytes, (CUstream)o.stream));
      CUevent e;
      if ((rc = record(&e, o.stream)) != ncclSuccess) return rc;
      p->read = e;
    }
    {
      std::lock_guard<std::mutex> lk(g->mu);
      p->bad = bad;
      p->consumed = true;
      g->cv.notify_all();
    }
    if (bad) rc = ncclInvalidUsage;
  }
  // 3) wait until every send has been consumed; the sender's stream then waits for the reader's copy
  size_t si = 0;
  for (const P2P& o : ops) {
    if (!o.send) continue;
    Group* g = sent[si].first;
    std::shared_ptr<Pending> p = sent[si++].second;
    {
      std::unique_lock<std::mutex> lk(g->mu);
      if (!wait(g, lk, [&] { return p->consumed; }, "a Recv matching a Send")) return ncclSystemError;
    }
    if (p->bad) { rc = ncclInvalidUsage; continue; }
    CU(cuStreamWaitEvent((CUstream)o.stream, p->read, 0));
    cuEventDestroy(p->read);
    cuEventDestroy(p->posted);
  }
  return rc;
}

template <class T>
void sum_into(void* acc, const void* v, size_t n) {
  T* a = static_cast<T*>(acc);
  const T* b = static_cast<const T*>(v);
  for (size_t i = 0; i < n; ++i) a[i] += b[i];
}

}  // namespace

extern "C" {

ncclResult_t ncclGetVersion(int* version) {
  if (!version) return ncclInvalidArgument;
  *version = NCCL_VERSION_CODE;
  return ncclSuccess;
}

const char* ncclGetErrorString(ncclResult_t r) {
  switch (r) {
    case ncclSuccess: return "no error (loopback)";
    case ncclUnhandledCudaError: return "unhandled cuda error (loopback)";
    case ncclSystemError: return "system error: a loopback rendezvous timed out";
    case ncclInternalError: return "internal error (loopback)";
    case ncclInvalidArgument: return "invalid argument (loopback)";
    case ncclInvalidUsage: return "invalid usage: ranks disagree on a collective (loopback)";
    default: return "unknown result (loopback)";
  }
}

ncclResult_t ncclGetUniqueId(ncclUniqueId* id) {
  if (!id) return ncclInvalidArgument;
  memset(id, 0, sizeof(*id));
  const uint64_t n = g_next_id++;
  snprintf(id->internal, sizeof(id->internal), "loopback:%llu", (unsigned long long)n);
  return ncclSuccess;
}

ncclResult_t ncclCommInitRank(ncclComm_t* comm, int nranks, ncclUniqueId id, int rank) {
  if (!comm) return ncclInvalidArgument;
  Comm* c = nullptr;
  const ncclResult_t r = init_rank(&c, nranks, std::string(id.internal, sizeof(id.internal)), rank);
  *comm = reinterpret_cast<ncclComm_t>(c);
  return r;
}

ncclResult_t ncclCommSplit(ncclComm_t comm, int color, int key, ncclComm_t* newcomm, ncclConfig_t*) {
  Comm* c = as_comm(comm);
  if (!c || !newcomm) return ncclInvalidArgument;
  *newcomm = nullptr;
  std::lock_guard<std::mutex> cl(c->mu);
  const uint64_t seq = c->calls++;
  Post mine;
  mine.op = OP_SPLIT; mine.color = color; mine.key = key;
  std::vector<Post> posts;
  ncclResult_t r = meet(c, seq, mine, posts);
  if (r == ncclSuccess && color != NCCL_SPLIT_NOCOLOR) {
    // ranks of this color, ordered by (key, parent rank)
    std::vector<std::pair<int, int>> members;
    for (int w = 0; w < c->world; ++w)
      if (posts[w].color == color) members.emplace_back(posts[w].key, w);
    std::sort(members.begin(), members.end());
    int nr = 0;
    for (size_t i = 0; i < members.size(); ++i)
      if (members[i].second == c->rank) nr = (int)i;
    const std::string k = c->g->key + "/split" + std::to_string(seq) + "/" + std::to_string(color);
    Comm* out = nullptr;
    r = init_rank(&out, (int)members.size(), k, nr);
    *newcomm = reinterpret_cast<ncclComm_t>(out);
  }
  leave(c, seq);
  return r;
}

ncclResult_t ncclCommDestroy(ncclComm_t comm) {
  Comm* c = as_comm(comm);
  if (!c) return ncclSuccess;
  Group* g = c->g;
  bool last;
  {
    std::lock_guard<std::mutex> lk(g->mu);
    last = --g->alive == 0;
  }
  if (last) {
    std::lock_guard<std::mutex> lk(g_reg_mu);
    g_reg.erase(g->key);
    delete g;
  }
  delete c;
  return ncclSuccess;
}

ncclResult_t ncclAllGather(const void* sendbuff, void* recvbuff, size_t sendcount, ncclDataType_t datatype, ncclComm_t comm,
                           cudaStream_t stream) {
  Comm* c = as_comm(comm);
  const size_t ts = type_size(datatype);
  if (!c || !ts) return ncclInvalidArgument;
  if (!ensure_ctx()) return ncclUnhandledCudaError;
  std::lock_guard<std::mutex> cl(c->mu);
  const uint64_t seq = c->calls++;
  const size_t bytes = sendcount * ts;
  Post mine;
  mine.op = OP_ALLGATHER; mine.count = sendcount; mine.dtype = datatype; mine.send = sendbuff; mine.recv = recvbuff;
  ncclResult_t r = record(&mine.posted, stream);
  if (r != ncclSuccess) return r;
  std::vector<Post> posts;
  r = meet(c, seq, mine, posts);
  CUevent read = nullptr;
  if (r == ncclSuccess) {
    for (int w = 0; w < c->world && r == ncclSuccess; ++w) {
      char* dst = static_cast<char*>(recvbuff) + (size_t)w * bytes;
      if (!bytes || (w == c->rank && posts[w].send == dst)) continue;  // in place: no self copy
      if (w != c->rank && !cu_ok(cuStreamWaitEvent((CUstream)stream, posts[w].posted, 0), "cuStreamWaitEvent")) r = ncclUnhandledCudaError;
      else if (!cu_ok(cuMemcpyAsync((CUdeviceptr)dst, (CUdeviceptr)posts[w].send, bytes, (CUstream)stream), "cuMemcpyAsync"))
        r = ncclUnhandledCudaError;
    }
    if (r == ncclSuccess) r = record(&read, stream);
    if (r == ncclSuccess) r = meet2(c, seq, read, posts);
    for (int w = 0; w < c->world && r == ncclSuccess; ++w)  // every peer read this rank's send buffer
      if (w != c->rank && !cu_ok(cuStreamWaitEvent((CUstream)stream, posts[w].read, 0), "cuStreamWaitEvent")) r = ncclUnhandledCudaError;
  }
  leave(c, seq);
  return r;
}

ncclResult_t ncclBroadcast(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t datatype, int root, ncclComm_t comm,
                           cudaStream_t stream) {
  Comm* c = as_comm(comm);
  const size_t ts = type_size(datatype);
  if (!c || !ts || root < 0 || root >= c->world) return ncclInvalidArgument;
  if (!ensure_ctx()) return ncclUnhandledCudaError;
  std::lock_guard<std::mutex> cl(c->mu);
  const uint64_t seq = c->calls++;
  const size_t bytes = count * ts;
  Post mine;
  mine.op = OP_BROADCAST; mine.count = count; mine.dtype = datatype; mine.root = root; mine.send = sendbuff; mine.recv = recvbuff;
  ncclResult_t r = record(&mine.posted, stream);
  if (r != ncclSuccess) return r;
  std::vector<Post> posts;
  r = meet(c, seq, mine, posts);
  if (r == ncclSuccess) {
    const Post& src = posts[root];
    if (bytes && src.send != recvbuff) {  // in place on the root: no self copy
      if (c->rank != root && !cu_ok(cuStreamWaitEvent((CUstream)stream, src.posted, 0), "cuStreamWaitEvent")) r = ncclUnhandledCudaError;
      else if (!cu_ok(cuMemcpyAsync((CUdeviceptr)recvbuff, (CUdeviceptr)src.send, bytes, (CUstream)stream), "cuMemcpyAsync"))
        r = ncclUnhandledCudaError;
    }
    CUevent read = nullptr;
    if (r == ncclSuccess) r = record(&read, stream);
    if (r == ncclSuccess) r = meet2(c, seq, read, posts);
    if (r == ncclSuccess && c->rank == root)
      for (int w = 0; w < c->world && r == ncclSuccess; ++w)
        if (w != root && !cu_ok(cuStreamWaitEvent((CUstream)stream, posts[w].read, 0), "cuStreamWaitEvent")) r = ncclUnhandledCudaError;
  }
  leave(c, seq);
  return r;
}

// Staged through the host: only the bulk-build plan uses it, and a sum in rank order is deterministic.
ncclResult_t ncclAllReduce(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t datatype, ncclRedOp_t op,
                           ncclComm_t comm, cudaStream_t stream) {
  Comm* c = as_comm(comm);
  if (!c) return ncclInvalidArgument;
  void (*add)(void*, const void*, size_t) = nullptr;
  switch (datatype) {
    case ncclInt32: add = sum_into<int32_t>; break;
    case ncclInt64: add = sum_into<int64_t>; break;
    case ncclUint64: add = sum_into<uint64_t>; break;
    case ncclFloat32: add = sum_into<float>; break;
    case ncclFloat64: add = sum_into<double>; break;
    default: break;
  }
  if (op != ncclSum || !add) {
    fprintf(stderr, "[nccl_loopback] AllReduce: only ncclSum over int32, int64, uint64, float32 and float64 is implemented\n");
    return ncclInvalidArgument;
  }
  if (!ensure_ctx()) return ncclUnhandledCudaError;
  std::lock_guard<std::mutex> cl(c->mu);
  const uint64_t seq = c->calls++;
  const size_t bytes = count * type_size(datatype);
  std::vector<char> host(bytes), acc(bytes, 0);
  CU(cuStreamSynchronize((CUstream)stream));
  if (bytes) CU(cuMemcpyDtoH(host.data(), (CUdeviceptr)sendbuff, bytes));
  Post mine;
  mine.op = OP_ALLREDUCE; mine.count = count; mine.dtype = datatype; mine.host = host.data();
  std::vector<Post> posts;
  ncclResult_t r = meet(c, seq, mine, posts);
  if (r == ncclSuccess) {
    for (int w = 0; w < c->world; ++w) add(acc.data(), posts[w].host, count);
    r = meet2(c, seq, nullptr, posts);  // every peer has read this rank's host values
  }
  if (r == ncclSuccess && bytes && !cu_ok(cuMemcpyHtoD((CUdeviceptr)recvbuff, acc.data(), bytes), "cuMemcpyHtoD")) r = ncclUnhandledCudaError;
  leave(c, seq);
  return r;
}

ncclResult_t ncclGroupStart() {
  ++t_depth;
  return ncclSuccess;
}

ncclResult_t ncclGroupEnd() {
  if (t_depth <= 0) return ncclInvalidUsage;
  if (--t_depth > 0) return ncclSuccess;
  std::vector<P2P> ops;
  ops.swap(t_ops);
  return run_group(std::move(ops));
}

static ncclResult_t p2p(bool send, void* buf, size_t count, ncclDataType_t datatype, int peer, ncclComm_t comm, cudaStream_t stream) {
  Comm* c = as_comm(comm);
  const size_t ts = type_size(datatype);
  if (!c || !ts || peer < 0 || peer >= c->world) return ncclInvalidArgument;
  t_ops.push_back(P2P{send, c, peer, buf, count * ts, stream});
  if (t_depth > 0) return ncclSuccess;
  std::vector<P2P> ops;
  ops.swap(t_ops);
  return run_group(std::move(ops));
}

ncclResult_t ncclSend(const void* sendbuff, size_t count, ncclDataType_t datatype, int peer, ncclComm_t comm, cudaStream_t stream) {
  return p2p(true, const_cast<void*>(sendbuff), count, datatype, peer, comm, stream);
}

ncclResult_t ncclRecv(void* recvbuff, size_t count, ncclDataType_t datatype, int peer, ncclComm_t comm, cudaStream_t stream) {
  return p2p(false, recvbuff, count, datatype, peer, comm, stream);
}

}  // extern "C"
