// shard.cu — list-sharded multi-GPU deployment behind the C ABI (b200vs_shard_*, include/b200vs.h).
//
// One process per GPU.  Every rank holds the replicated trained state (centroids; IVF-PQ: and codebooks) of ONE logical
// IVF-Flat or IVF-PQ index and the rows of the inverted lists it owns (contiguous blocks of lists per rank — equivalently
// Raft regions mapped to GPUs, src/vector/vector_index.h:54-55).  A batched search is:
//   1. coarse quantiser on this rank's SLICE of the batch (all ranks hold all queries), one all-gather of the probe table
//      (the faiss quantizer->search step of IndexIVF::search, src/vector/vector_index_ivf_flat.cc:247-251);
//   2. scan of the probed lists this rank owns (IVF-Flat: the tile scan, csrc/tc_scan.cu; IVF-PQ: the LUT scan, with the
//      coarse value of every probe recomputed on the rank, csrc/ivf_pq.cu) -> exact local top-k;
//   3. ONE ncclAllGather of the packed per-shard top-k ((distance, id) 16-byte records) over NVLink, then the k-way merge
//      kernel — the engine's analogue of VectorIndexWrapper::MergeSearchResults (src/vector/vector_index.cc:1056-1108).
// FLAT and HNSW shard by row instead (DESIGN.md 4.5): row id lives on rank row_owner_of(id), each rank holds a standalone
// index of its rows, and a search skips step 1 and runs the whole batch on the rank's index before the same all-gather + merge.
// The binary types take the same two routes through the b200vs_shard_*_binary entry points: BINARY_IVF_FLAT by list (Hamming
// coarse pass, binary list scan), BINARY_FLAT by row.  Rows and queries then travel as packed bits, dim / 8 bytes each, and
// the merge key is the Hamming distance itself.
// Both kinds share one write path: b200vs_shard_add* partitions the rows by owner on the device (list-sharded: the owner of
// the list the sender assigns the row to), moves them with one grouped ncclSend/ncclRecv, and every rank returns the first
// refusal in rank order or adds.  A world of one runs the same code with only the NCCL calls left out.
//
// NCCL is resolved at run time (dlopen of libnccl.so.2): a single-GPU dingo-store node needs no NCCL at all, and a process
// that already carries an NCCL (e.g. the one bundled with PyTorch in the test harness) shares it.  Each in-flight lane owns
// its communicator (ncclCommSplit), so batches in flight overlap across streams; callers order batches with a sequence
// number, which maps every batch to the same communicator on every rank.
#include <dlfcn.h>
#include <nccl.h>
#include <unistd.h>

#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <memory>
#include <vector>

#include "index.h"
#include "ivf_common.h"

namespace b200vs {

// ---------------------------------------------------------------------------------------------
// NCCL, resolved lazily
// ---------------------------------------------------------------------------------------------
struct NcclApi {
  void* h = nullptr;
  decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
  decltype(&ncclCommInitRank) CommInitRank = nullptr;
  decltype(&ncclCommSplit) CommSplit = nullptr;
  decltype(&ncclCommDestroy) CommDestroy = nullptr;
  decltype(&ncclAllGather) AllGather = nullptr;
  decltype(&ncclAllReduce) AllReduce = nullptr;
  decltype(&ncclBroadcast) Broadcast = nullptr;
  decltype(&ncclSend) Send = nullptr;
  decltype(&ncclRecv) Recv = nullptr;
  decltype(&ncclGroupStart) GroupStart = nullptr;
  decltype(&ncclGroupEnd) GroupEnd = nullptr;
  decltype(&ncclGetErrorString) GetErrorString = nullptr;
  decltype(&ncclGetVersion) GetVersion = nullptr;
};

static NcclApi& nccl() {
  static NcclApi api;
  static std::mutex mu;
  std::lock_guard<std::mutex> g(mu);
  if (api.h) return api;
  const char* env = getenv("B200VS_NCCL_LIB");
  const char* names[] = {env, "libnccl.so.2", "libnccl.so"};
  void* h = nullptr;
  for (const char* n : names) {
    if (!n || !*n) continue;
    h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (h) break;
  }
  if (!h) fail(B200VS_EVECTOR_NOT_SUPPORT, "NCCL not found (libnccl.so.2): list-sharded search needs it; set B200VS_NCCL_LIB");
#define B200VS_SYM(field, name)                                                                 \
  api.field = reinterpret_cast<decltype(api.field)>(dlsym(h, name));                            \
  if (!api.field) fail(B200VS_EVECTOR_NOT_SUPPORT, std::string("NCCL symbol missing: ") + name)
  B200VS_SYM(GetUniqueId, "ncclGetUniqueId");
  B200VS_SYM(CommInitRank, "ncclCommInitRank");
  B200VS_SYM(CommSplit, "ncclCommSplit");
  B200VS_SYM(CommDestroy, "ncclCommDestroy");
  B200VS_SYM(AllGather, "ncclAllGather");
  B200VS_SYM(AllReduce, "ncclAllReduce");
  B200VS_SYM(Broadcast, "ncclBroadcast");
  B200VS_SYM(Send, "ncclSend");
  B200VS_SYM(Recv, "ncclRecv");
  B200VS_SYM(GroupStart, "ncclGroupStart");
  B200VS_SYM(GroupEnd, "ncclGroupEnd");
  B200VS_SYM(GetErrorString, "ncclGetErrorString");
  B200VS_SYM(GetVersion, "ncclGetVersion");
#undef B200VS_SYM
  api.h = h;
  return api;
}

#define B200VS_NCCL(expr)                                                                                          \
  do {                                                                                                             \
    ncclResult_t _r = (expr);                                                                                      \
    if (_r != ncclSuccess && _r != ncclInProgress)                                                                 \
      fail(B200VS_EINTERNAL, std::string(#expr) + " failed: " + nccl().GetErrorString(_r));                        \
  } while (0)

// ---------------------------------------------------------------------------------------------
// kernels: pack / merge of 16-byte (distance, id) records, owner routing
// ---------------------------------------------------------------------------------------------
struct __align__(16) TopkRec {
  float dist;
  int pad;
  long long id;
};
static_assert(sizeof(TopkRec) == 16, "one 16-byte record per hit");

static __global__ void pack_topk_kernel(const float* __restrict__ d, const long long* __restrict__ id, long long n, TopkRec* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  TopkRec r;
  r.dist = d[i]; r.pad = 0; r.id = id[i];
  out[i] = r;
}

// parts [world, nq, k] records (ascending per part, id < 0 = empty) -> merged [nq, k]: (distance, id) ascending.
// One warp per query: world * k <= 1024 records, each lane ranks its records against all others... for the usual
// world * k <= 256 a rank sort in shared memory is cheapest.
constexpr int MERGE_WARPS = 4;
constexpr int MERGE_MAX = 256;
static __global__ void __launch_bounds__(MERGE_WARPS * 32)
merge_packed_warp_kernel(const TopkRec* __restrict__ parts, int world, long long nq, int k, float* out_dist, long long* out_ids) {
  __shared__ uint32_t s_kd[MERGE_WARPS][MERGE_MAX];
  __shared__ long long s_id[MERGE_WARPS][MERGE_MAX];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long q = (long long)blockIdx.x * MERGE_WARPS + warp;
  if (q >= nq) return;
  const int tot = world * k;
  int m = 0;
  for (int base = 0; base < tot; base += 32) {
    const int i = base + lane;
    TopkRec r;
    r.id = -1; r.dist = 0.f;
    if (i < tot) r = parts[((size_t)(i / k) * nq + q) * k + (i % k)];
    const bool ok = r.id >= 0;
    const unsigned msk = __ballot_sync(0xffffffffu, ok);
    if (ok) { const int p = m + __popc(msk & ((1u << lane) - 1u)); s_kd[warp][p] = f2ord(r.dist); s_id[warp][p] = r.id; }
    m += __popc(msk);
  }
  __syncwarp();
  for (int e = lane; e < m; e += 32) {
    const uint32_t d0 = s_kd[warp][e];
    const long long i0 = s_id[warp][e];
    int rank = 0;
    for (int j = 0; j < m; ++j) {
      const uint32_t dj = s_kd[warp][j];
      const long long ij = s_id[warp][j];
      rank += (key_less(dj, ij, d0, i0) || (dj == d0 && ij == i0 && j < e)) ? 1 : 0;
    }
    if (rank < k) { out_dist[(size_t)q * k + rank] = ord2f(d0); out_ids[(size_t)q * k + rank] = i0; }
  }
  for (int i = min(m, k) + lane; i < k; i += 32) { out_dist[(size_t)q * k + i] = 0.f; out_ids[(size_t)q * k + i] = -1; }
}

// One round of the deep merge's pairwise tree: runs in [nruns, nqc, k], each ascending by (f2ord(key), id) with id < 0
// padding at its tail; run i of the output [cdiv(nruns, 2), nqc, k] is the first k records of runs (2i, 2i + 1) in
// (f2ord(key), id, run) order (a last run without a partner is copied).  Record j of a run lands at j + its rank in the
// partner run: a lower bound from the left run, an upper bound from the right one, so equal records keep run order, every
// output slot is written once and the padding lands at the tail.  A record that cannot land below k stops its search at
// k - j.  FINAL: the output is the last round's single run, written as (distance, id) into od / oi [nqc, k] with -1 / 0 padding.
// Grid (cdiv(k, MERGE_RUN_THREADS), cdiv(nruns, 2), nqc).
constexpr int MERGE_RUN_THREADS = 256;
__device__ __forceinline__ bool rec_less(const TopkRec& a, const TopkRec& b) {  // padding after every record
  if (a.id < 0) return false;
  if (b.id < 0) return true;
  return key_less(f2ord(a.dist), a.id, f2ord(b.dist), b.id);
}
template <bool FINAL>
static __global__ void __launch_bounds__(MERGE_RUN_THREADS)
merge_runs_kernel(const TopkRec* __restrict__ in, int nruns, int nqc, int k, TopkRec* out, float* od, long long* oi) {
  const int j = blockIdx.x * MERGE_RUN_THREADS + threadIdx.x;
  if (j >= k) return;
  const int pair = blockIdx.y, q = blockIdx.z;
  const TopkRec* a = in + ((size_t)(2 * pair) * nqc + q) * k;
  const TopkRec* b = a + (size_t)nqc * k;
  const bool has_b = 2 * pair + 1 < nruns;
  const size_t o = ((size_t)pair * nqc + q) * k;
  auto emit = [&](int pos, TopkRec r) {
    if (pos >= k) return;
    if (r.id < 0) { r.dist = 0.f; r.id = -1; }
    if (FINAL) { od[o + pos] = r.dist; oi[o + pos] = r.id; }
    else out[o + pos] = r;
  };
  const TopkRec ra = a[j];
  if (!has_b) { emit(j, ra); return; }
  int lo = 0, hi = k - j;  // a[j]: the records of b strictly before it
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (rec_less(b[mid], ra)) lo = mid + 1; else hi = mid;
  }
  emit(j + lo, ra);
  const TopkRec rb = b[j];
  lo = 0; hi = k - j;  // b[j]: the records of a not after it
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (!rec_less(rb, a[mid])) lo = mid + 1; else hi = mid;
  }
  emit(j + lo, rb);
}

static __global__ void unpack_parts_kernel(const TopkRec* __restrict__ parts, long long n, float* d, long long* id) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const TopkRec r = parts[i];
  d[i] = r.dist; id[i] = r.id;
}

// The finish of a merged read [nq, k] (merge_key in the read section): ip = 1, the merged key -ip -> the API distance 1 - ip,
// rounded as the single-index finish rounds it; counts (range, else null): counts[q] = merged rows of query q (the rows are
// ascending with -1 padding at the end).
static __global__ void merge_finish_kernel(float* dist, const long long* __restrict__ ids, long long nq, int k, int ip, int* counts) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq * k) return;
  const int j = (int)(i % k);
  const bool hit = ids[i] >= 0;
  if (hit && ip) dist[i] = __fsub_rn(1.0f, -dist[i]);
  if (counts && (hit ? (j == k - 1 || ids[i + 1] < 0) : j == 0)) counts[i / k] = hit ? j + 1 : 0;
}

static __global__ void fill_ll_kernel(long long* p, long long n, long long v) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

static __global__ void count_lists_kernel(const long long* __restrict__ lists, long long n, int nlist, unsigned long long* counts) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { const long long l = lists[i]; if (l >= 0 && l < nlist) atomicAdd(counts + l, 1ULL); }
}

constexpr int ROUTE_MAX_WORLD = 1024;  // ranks of a sharded index (the routing kernels' shared-memory table)

// The owner of a row of a row-sharded (FLAT / HNSW) index: splitmix64's finalizer of the id read as a uint64, mod world.
// The one definition for the host (b200vs_row_owner) and the device (row routing).  z mod world is taken 16 bits at a
// time in 32-bit arithmetic, exact for world <= ROUTE_MAX_WORLD (each partial value stays below 2^26), which keeps the
// 64-bit division routine out of the routing kernels.
__host__ __device__ __forceinline__ int row_owner_of(long long id, int world) {
  unsigned long long z = (unsigned long long)id;
  z ^= z >> 30;
  z *= 0xbf58476d1ce4e5b9ULL;
  z ^= z >> 27;
  z *= 0x94d049bb133111ebULL;
  z ^= z >> 31;
  const unsigned w = (unsigned)world, lo = (unsigned)z;
  unsigned r = (unsigned)(z >> 32) % w;
  r = ((r << 16) | (lo >> 16)) % w;
  r = ((r << 16) | (lo & 0xffffu)) % w;
  return (int)r;
}

// Stable partition of rows by owner, in tiles of ROUTE_THREADS rows: route_count_kernel counts each tile's rows per owner
// into an owner-major table cnt[owner * ntiles + tile], route_offsets_kernel scans that table (its exclusive prefix sum is
// the first output slot of every (owner, tile)), and route_scatter_kernel moves each row to its slot, so each owner's rows
// keep the caller's order.
constexpr int ROUTE_THREADS = 256, ROUTE_WARPS = ROUTE_THREADS / 32;  // s_cnt below: ROUTE_WARPS * world ints of shared memory
constexpr int ROUTE_SCAN_THREADS = 1024;

// The owner rules of the routing kernels, applied to a row's key.  Row-sharded: the key is the id.  List-sharded: the key is
// the row's inverted list, which travels with the row; rank r owns the lists [r * per, (r + 1) * per), per = ceil(nlist / W).
struct RowOwner {
  static constexpr bool kLists = false;
  __device__ __forceinline__ int operator()(long long id, int W) const { return row_owner_of(id, W); }
};
struct ListOwner {
  static constexpr bool kLists = true;
  int per;
  __device__ __forceinline__ int operator()(long long list, int) const { return (int)list / per; }
};

// This thread's row of the tile: returns (its owner, -1 past n; the rows of that owner before it in its warp), and
// s_cnt[warp * W + owner] = the warp's rows of that owner.
template <class Owner>
static __device__ __forceinline__ int2 route_tile(const long long* __restrict__ keys, long long n, int W, Owner owner, int* s_cnt) {
  for (int i = threadIdx.x; i < ROUTE_WARPS * W; i += ROUTE_THREADS) s_cnt[i] = 0;
  __syncthreads();
  const long long i = (long long)blockIdx.x * ROUTE_THREADS + threadIdx.x;
  const int o = i < n ? owner(keys[i], W) : -1;
  const unsigned peers = __match_any_sync(0xffffffffu, o);
  const int lane = threadIdx.x & 31;
  if (o >= 0 && __ffs(peers) - 1 == lane) s_cnt[(threadIdx.x >> 5) * W + o] = __popc(peers);
  __syncthreads();
  return make_int2(o, __popc(peers & ((1u << lane) - 1u)));
}

template <class Owner>
static __global__ void __launch_bounds__(ROUTE_THREADS) route_count_kernel(const long long* __restrict__ keys, long long n, int W, Owner owner, int* cnt) {
  extern __shared__ int s_cnt[];
  route_tile(keys, n, W, owner, s_cnt);
  for (int o = threadIdx.x; o < W; o += ROUTE_THREADS) {
    int c = 0;
    for (int w = 0; w < ROUTE_WARPS; ++w) c += s_cnt[w * W + o];
    cnt[(size_t)o * gridDim.x + blockIdx.x] = c;
  }
}

// One CTA: off[i] = sum of cnt[0, i) over the m = W * ntiles entries, in chunks of ROUTE_SCAN_THREADS (a warp-shuffle scan,
// one scan of the warp totals, a running carry); owner_cnt[o] = rows of owner o.
static __global__ void __launch_bounds__(ROUTE_SCAN_THREADS)
route_offsets_kernel(const int* __restrict__ cnt, long long ntiles, int W, long long* off, long long* owner_cnt) {
  __shared__ long long s_warp[ROUTE_SCAN_THREADS / 32];
  __shared__ long long s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long m = ntiles * W;
  if (threadIdx.x == 0) s_carry = 0;
  for (long long base = 0; base < m; base += ROUTE_SCAN_THREADS) {
    const long long i = base + threadIdx.x;
    const long long v = i < m ? cnt[i] : 0;
    long long x = v;
    for (int sh = 1; sh < 32; sh <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, x, sh);
      if (lane >= sh) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
      long long w = s_warp[lane];
      for (int sh = 1; sh < 32; sh <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, w, sh);
        if (lane >= sh) w += y;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    const long long incl = s_carry + (warp ? s_warp[warp - 1] : 0) + x;
    if (i < m) off[i] = incl - v;
    __syncthreads();
    if (threadIdx.x == ROUTE_SCAN_THREADS - 1) s_carry = incl;
  }
  __syncthreads();
  for (int o = threadIdx.x; o < W; o += ROUTE_SCAN_THREADS)
    owner_cnt[o] = (o + 1 < W ? off[(o + 1) * ntiles] : s_carry) - off[o * ntiles];
}

// moves rows, ids and (Owner::kLists) lists to their slots.  A row is rb opaque bytes (FP32 rows: 4 * d; IVF-PQ: the
// stored code row), moved 16, 4 or 1 bytes at a time as the row size and the two base addresses allow.
template <class Owner>
static __global__ void __launch_bounds__(ROUTE_THREADS)
route_scatter_kernel(const unsigned char* __restrict__ x, const long long* __restrict__ ids, const long long* __restrict__ lists, long long n,
                     int rb, int W, Owner owner, const long long* __restrict__ off, unsigned char* ox, long long* oids, long long* olists) {
  extern __shared__ int s_cnt[];
  __shared__ long long s_dst[ROUTE_THREADS];
  const int2 t = route_tile(Owner::kLists ? lists : ids, n, W, owner, s_cnt);
  const int o = t.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (o >= 0) {
    long long p = off[(size_t)o * gridDim.x + blockIdx.x] + t.y;
    for (int w = 0; w < warp; ++w) p += s_cnt[w * W + o];
    s_dst[threadIdx.x] = p;
  }
  __syncthreads();
  const long long r0 = (long long)blockIdx.x * ROUTE_THREADS;
  const size_t base = reinterpret_cast<size_t>(x) | reinterpret_cast<size_t>(ox);
  const int width = (rb & 15) == 0 && (base & 15) == 0 ? 16 : (rb & 3) == 0 && (base & 3) == 0 ? 4 : 1;
  for (int j = warp; j < ROUTE_THREADS && r0 + j < n; j += ROUTE_WARPS) {  // one warp per row
    const long long src = r0 + j, dst = s_dst[j];
    const unsigned char* xs = x + (size_t)src * rb;
    unsigned char* xd = ox + (size_t)dst * rb;
    if (width == 16) {
#pragma unroll 1
      for (int i = lane; i < (rb >> 4); i += 32) reinterpret_cast<uint4*>(xd)[i] = reinterpret_cast<const uint4*>(xs)[i];
    } else if (width == 4) {
      for (int i = lane; i < (rb >> 2); i += 32) reinterpret_cast<uint32_t*>(xd)[i] = reinterpret_cast<const uint32_t*>(xs)[i];
    } else {
      for (int i = lane; i < rb; i += 32) xd[i] = xs[i];
    }
    if (lane == 0) {
      oids[dst] = ids[src];
      if (Owner::kLists) olists[dst] = lists[src];
    }
  }
}

// Restore of a list-major rank file: out[i] = the list holding row r0 + i, off[nlist + 1] being the file's list offsets
// (ascending; the last list wins an empty-list tie, as the rows of a list start at its offset).
static __global__ void expand_lists_kernel(const long long* __restrict__ off, int nlist, long long r0, long long n, long long* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long row = r0 + i;
  int lo = 0, hi = nlist - 1;  // the largest l with off[l] <= row
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= row) lo = mid;
    else hi = mid - 1;
  }
  out[i] = lo;
}

// Rows of a restored rank file that the owner rule does not give to `rank`, counted into *bad (the tile shape of
// route_count_kernel, with the same Owner functors).
template <class Owner>
static __global__ void __launch_bounds__(ROUTE_THREADS)
owner_check_kernel(const long long* __restrict__ keys, long long n, int W, Owner owner, int rank, unsigned long long* bad) {
  const long long i = (long long)blockIdx.x * ROUTE_THREADS + threadIdx.x;
  const bool off_rank = i < n && owner(keys[i], W) != rank;
  const unsigned msk = __ballot_sync(0xffffffffu, off_rank);
  if ((threadIdx.x & 31) == 0 && msk) atomicAdd(bad, (unsigned long long)__popc(msk));
}

// The write gate of a set (b200vs_shard::add_mu): its writes (add, delete, train, state broadcast, save, load, the rule, a
// rebuild INTO it) hold it exclusively, one at a time; a rebuild that reads the set holds it shared.  A shared hold is granted
// whenever no exclusive one is held, even while a writer waits: two rebuilds that read one set (a split's child and parent)
// never wait for each other's locks, whatever order they start in on each rank.  Their collectives are not ordered by the
// gate (include/b200vs.h states the caller's rule on NCCL).
struct Gate {
  std::mutex mu;
  std::condition_variable cv;
  int readers = 0;
  bool writer = false;
  void lock() {
    std::unique_lock<std::mutex> lk(mu);
    cv.wait(lk, [&] { return !writer && readers == 0; });
    writer = true;
  }
  void unlock() {
    { std::lock_guard<std::mutex> lk(mu); writer = false; }
    cv.notify_all();
  }
  void lock_shared() {
    std::unique_lock<std::mutex> lk(mu);
    cv.wait(lk, [&] { return !writer; });
    ++readers;
  }
  void unlock_shared() {
    { std::lock_guard<std::mutex> lk(mu); --readers; }
    cv.notify_all();
  }
};

}  // namespace b200vs

using namespace b200vs;

// ---------------------------------------------------------------------------------------------
// the shard handle
// ---------------------------------------------------------------------------------------------
struct b200vs_shard {
  IndexBase* ix = nullptr;
  int rank = 0, world = 1, nlanes = 1;
  bool rows = false;  // sharded by rows (shard_by_rows: owner(id) = row_owner_of), else by inverted list (shard_by_lists)
  struct SLane {
    ncclComm_t comm = nullptr;
    std::mutex mu;
    DevBuf<long long> probes;   // [per * world, nprobe]
    DevBuf<TopkRec> parts;      // [world, nq, k]
    DevBuf<unsigned char> q_all;  // host-pointer variant: [per * world] query rows of query_row_bytes()
    DevBuf<float> od;           // local / merged results
    DevBuf<long long> oi;
    cudaStream_t own = nullptr;
    cudaStream_t last = nullptr;  // stream of the lane's previous batch
    cudaEvent_t done = nullptr;   // recorded behind it: a batch on another stream waits for it before touching the buffers
  };
  std::vector<std::unique_ptr<SLane>> lanes;
  std::mutex seq_mu;
  std::condition_variable seq_cv;
  int64_t next_auto = 0;             // sequence numbers handed out when the caller passes seq < 0
  int64_t next_seq = 0;              // the batch whose turn it is to be enqueued
  // write path (collective, one at a time; rebuilds that read this set hold the gate shared)
  Gate add_mu;
  cudaStream_t ws = nullptr;
  DevBuf<unsigned long long> plan_counts;  // [nlist] rows per list seen by b200vs_shard_plan_add*
  bool planning = false;
  // the training size of b200vs_shard_need_rebuild's rule for the whole set (list-sharded): the rows shard_train clustered
  // over every rank, or every rank's live rows summed at shard_broadcast_state / shard_load; not saved, as on one index
  int64_t train_rows_set = 0;

  ~b200vs_shard() {
    if (ix) cudaSetDevice(ix->device);
    for (auto& l : lanes) {
      if (l->own) { cudaStreamSynchronize(l->own); cudaStreamDestroy(l->own); }
      if (l->done) { cudaEventSynchronize(l->done); cudaEventDestroy(l->done); }
      if (l->comm) nccl().CommDestroy(l->comm);
    }
    if (ws) { cudaStreamSynchronize(ws); cudaStreamDestroy(ws); }
  }
  int lists_per_rank() const { return (ix->nlist_now() + world - 1) / world; }
};

namespace {

// The two ways an index type is sharded, each decided here only: by row (owner(id) = row_owner_of) or by inverted list
bool shard_by_rows(b200vs_type t) { return t == B200VS_FLAT || t == B200VS_HNSW || t == B200VS_BINARY_FLAT; }
bool shard_by_lists(b200vs_type t) { return t == B200VS_IVF_FLAT || t == B200VS_IVF_PQ || t == B200VS_BINARY_IVF_FLAT; }

b200vs_shard* get(b200vs_shard* s) {
  if (!s || !s->ix) fail(B200VS_EILLEGAL_PARAMETERS, "null shard handle");
  return s;
}

// the float data calls on a binary shard, and the b200vs_shard_*_binary ones on a float shard
void check_row_type(const b200vs_shard* sh, bool binary_call) {
  if (sh->ix->binary() != binary_call)
    fail(B200VS_EILLEGAL_PARAMETERS, binary_call ? "binary entry point on a float shard" : "float entry point on a binary shard");
}

// Take the turn of batch `seq` (seq < 0: the next one in call order).  Batches are ENQUEUED strictly in sequence order on
// every rank (the enqueue is asynchronous, so batches still overlap on the GPU): a device-wide synchronisation hidden in
// one batch's enqueue (cudaFree / cudaMalloc of a growing buffer) then only ever waits for kernels of earlier batches,
// which every rank has already enqueued — enqueueing two communicators' collectives in different orders on different ranks
// is the classic multi-communicator deadlock.  Batch seq uses lane / communicator seq % nlanes.
struct SeqLane {
  b200vs_shard* sh;
  b200vs_shard::SLane* lane;
  int64_t seq;
  SeqLane(b200vs_shard* s, int64_t seq_) : sh(s), seq(seq_) {
    std::unique_lock<std::mutex> lk(sh->seq_mu);
    if (seq < 0) seq = sh->next_auto;
    sh->next_auto = std::max(sh->next_auto, seq + 1);
    if (seq < sh->next_seq) fail(B200VS_EILLEGAL_PARAMETERS, "shard search: sequence number already used");
    sh->seq_cv.wait(lk, [&] { return sh->next_seq == seq; });
    lane = sh->lanes[(size_t)(seq % sh->nlanes)].get();
    lane->mu.lock();
  }
  ~SeqLane() {
    lane->mu.unlock();
    {
      std::lock_guard<std::mutex> lk(sh->seq_mu);
      sh->next_seq = seq + 1;
    }
    sh->seq_cv.notify_all();
  }
};

// All-gathers `count` host values of every rank through the write stream: returns [world, count], rank r's at r * count.
template <class T>
std::vector<T> all_gather_host(b200vs_shard* sh, const T* mine, size_t count = 1) {
  const int W = sh->world;
  std::vector<T> all((size_t)W * count);
  DevBuf<T> buf;
  buf.reserve((size_t)W * count, 0, sh->ws);
  T* slot = buf.p + (size_t)sh->rank * count;
  B200VS_CUDA(cudaMemcpyAsync(slot, mine, count * sizeof(T), cudaMemcpyHostToDevice, sh->ws));
  if (W > 1) B200VS_NCCL(nccl().AllGather(slot, buf.p, count * sizeof(T), ncclUint8, sh->lanes[0]->comm, sh->ws));
  B200VS_CUDA(cudaMemcpyAsync(all.data(), buf.p, all.size() * sizeof(T), cudaMemcpyDeviceToHost, sh->ws));
  B200VS_CUDA(cudaStreamSynchronize(sh->ws));
  return all;
}

// Status agreement of a collective step: attempt(f) runs this rank's part and keeps its status, agree() all-gathers the
// statuses and returns the first failure in rank order (OK when every rank succeeded), the same on every rank.
struct Status {
  int code = B200VS_OK;
  std::string msg;
};
template <class F>
Status attempt(F&& f) {
  Status st;
  st.code = guarded([&]() -> int { f(); return B200VS_OK; });
  if (st.code != B200VS_OK) st.msg = g_last_error;
  return st;
}
Status agree(b200vs_shard* sh, const Status& mine, const char* what) {
  const std::vector<int> codes = all_gather_host(sh, &mine.code);
  for (int w = 0; w < sh->world; ++w)
    if (codes[w] != B200VS_OK) return Status{codes[w], w == sh->rank ? mine.msg : std::string(what) + " refused by rank " + std::to_string(w)};
  return Status{};
}
void check(const Status& st) {
  if (st.code != B200VS_OK) fail(st.code, st.msg);
}
// A local step of a collective call (allocations, kernels, an index write) that the next collective depends on.  agreed:
// every rank's status is agreed after it, so a device failure on one rank (an allocation that does not fit) is returned by
// every rank instead of leaving its peers waiting in that collective.  Else f runs as it is.
template <class F>
void local_step(b200vs_shard* sh, bool agreed, const char* what, F&& f) {
  if (agreed) check(agree(sh, attempt(f), what));
  else f();
}

// One sharded read, as its extern "C" entry point passes it.  k: results per query (range: max_results).  on_device: xq and
// the outputs are device pointers and the read runs on `stream` (null: the lane's own stream); else they are host pointers,
// every rank passes the SAME batch (upload_batch), and the call returns with the results on the host.
enum ReadKind { READ_TOPK, READ_DEEP, READ_RANGE };
struct ShardRead {
  ReadKind kind;
  bool binary_call;  // a b200vs_shard_*_binary* entry point: packed queries
  bool on_device;
  void* stream;
  int64_t seq, nq;
  const void* xq;
  float radius;  // range
  int k;
  const b200vs_search_params* sp;
  float* od;
  int64_t* oi;
  int32_t* oc;   // range: merged rows per query
};

// The merge key rule of every sharded read (the table of DESIGN.md 4.5): what each rank's results are keyed on for the pack
// and the merge, and what merge_finish_kernel does to the merged key.  The single-index select ranks IP / cosine hits by
// -ip, and two distinct inner products can round to the same 1 - ip (near ip = 2^-10 the spacing of ip is 2^-34 and that of
// 1 - ip 2^-24), which a merge on the API distance would choose and order by id.  So the reads that equal their single-index
// call bit for bit (row-sharded FLAT top-k, deep on the float types, range) ask for the raw value (raw), negate ip to -ip
// before the pack and form 1 - ip after the merge with the single index's own __fsub_rn (neg).  The list-sharded float
// top-k keeps the API distance: it merges by MergeSearchResults' rule (the regions' results on the distance they return),
// and another key would change which of two such rows it returns.  HNSW keys on hnsw_distance (L2 distance | 1 - ip), the
// distance its walk ranks by; its search refuses raw.  The Hamming distance is exact and is the API distance.
struct MergeKey { bool raw, neg; };
MergeKey merge_key(const b200vs_shard* sh, ReadKind kind) {
  const IndexBase* ix = sh->ix;
  const bool raw = kind == READ_RANGE || (kind == READ_DEEP && !ix->binary()) || (sh->rows && ix->type == B200VS_FLAT);
  return {raw, raw && ix->ip_like()};  // a binary index's metric is Hamming
}

// Step 3 of a sharded read: the per-shard results L.od / L.oi [nq, k] are packed into 16-byte records, all-gathered and
// merged into out_* [nq, k], one query chunk at a time.  Top-k and range: the whole batch is one chunk, so ONE all-gather.
// Deep, whose k is bounded by kDeepMaxK and not by shared memory: nqc queries per chunk from (W, k, nq) alone so that every
// rank agrees, with the gathered records W * nqc * k * 16 B within the deep path's 1 GiB budget (W = 8, k = 40960: 204
// queries).  The merge of a chunk: deep, ceil(log2 W) rounds of merge_runs_kernel (one copy round when W = 1), ping-ponging
// between L.parts and a scratch buffer of ceil(W / 2) runs when W > 2; else the warp merge when W * k <= MERGE_MAX, or
// unpack and the block merge.
void gather_merge(b200vs_shard* sh, b200vs_shard::SLane& L, int64_t nq, int k, bool deep, float* out_dist, long long* out_ids,
                  cudaStream_t s) {
  IndexBase* ix = sh->ix;
  const int W = sh->world, r = sh->rank;
  const long long run_bytes = (long long)W * k * (long long)sizeof(TopkRec);
  const int64_t nqc_max = deep ? std::max<int64_t>(1, std::min<int64_t>({nq, (1LL << 30) / run_bytes, 65535})) : nq;
  L.parts.reserve((size_t)W * nqc_max * k, 0, s);
  TopkRec* tmp = deep && W > 2 ? ix->scratch.alloc<TopkRec>((size_t)((W + 1) / 2) * nqc_max * k) : nullptr;  // W <= 2: one final round
  for (int64_t q0 = 0; q0 < nq; q0 += nqc_max) {
    const int64_t nqc = std::min<int64_t>(nqc_max, nq - q0);
    const long long nk = (long long)nqc * k;
    float* od = out_dist + (size_t)q0 * k;
    long long* oi = out_ids + (size_t)q0 * k;
    ix->phase(IndexBase::PH_MERGE, s);
    pack_topk_kernel<<<(unsigned)cdiv(nk, 256), 256, 0, s>>>(L.od.p + (size_t)q0 * k, L.oi.p + (size_t)q0 * k, nk, L.parts.p + (size_t)r * nk);
    ix->phase(IndexBase::PH_COMM, s);
    if (W > 1) B200VS_NCCL(nccl().AllGather(L.parts.p + (size_t)r * nk, L.parts.p, (size_t)nk * sizeof(TopkRec), ncclUint8, L.comm, s));
    ix->phase(IndexBase::PH_MERGE, s);
    int launches = 3;  // b200vs_last_search_stats[0]: 3 for a top-k or range merge, whichever kernels it takes
    if (deep) {  // the pack, the rounds of more than one pair, the final round into out_*
      const unsigned kb = (unsigned)cdiv(k, MERGE_RUN_THREADS);
      const TopkRec* in = L.parts.p;
      int runs = W;
      for (launches = 2; runs > 2; runs = (runs + 1) / 2, ++launches) {
        TopkRec* out = in == L.parts.p ? tmp : L.parts.p;
        merge_runs_kernel<false><<<dim3(kb, (runs + 1) / 2, (unsigned)nqc), MERGE_RUN_THREADS, 0, s>>>(in, runs, (int)nqc, k, out, nullptr, nullptr);
        in = out;
      }
      merge_runs_kernel<true><<<dim3(kb, 1, (unsigned)nqc), MERGE_RUN_THREADS, 0, s>>>(in, runs, (int)nqc, k, nullptr, od, oi);
    } else if (W * k <= MERGE_MAX) {
      merge_packed_warp_kernel<<<(unsigned)cdiv(nqc, MERGE_WARPS), MERGE_WARPS * 32, 0, s>>>(L.parts.p, W, nqc, k, od, oi);
    } else {  // wide merges: unpack and use the block merge kernel
      float* pd = ix->scratch.alloc<float>((size_t)W * nk);
      long long* pi = ix->scratch.alloc<long long>((size_t)W * nk);
      unpack_parts_kernel<<<(unsigned)cdiv(W * nk, 256), 256, 0, s>>>(L.parts.p, W * nk, pd, pi);
      launch_merge_api(W, nqc, k, pd, pi, od, oi, s);
    }
    B200VS_CUDA(cudaGetLastError());
    ix->launch_count(launches);
  }
  ix->phase(IndexBase::PH_OTHER, s);
}

// The flow of a sharded read: queries (all nq of them, raw) are on the device in `xq`; merged results land in out_* (device;
// out_counts: range only) on stream s.  Step 2 is this rank's one search request, keyed by merge_key, into L.od / L.oi:
// ascending, -1-padded [nq, k] (key, id) lists.  List-sharded: it searches the prepared queries over the gathered probe
// table L.probes.  Row-sharded: there is no coarse step, and it searches the raw queries (the rank's index prepares them).
// Queries are rows of query_row_bytes(): FP32, or packed bits on a binary index.
void shard_stream(b200vs_shard* sh, b200vs_shard::SLane& L, const ShardRead& rd, const void* xq, float* out_dist, long long* out_ids,
                  int* out_counts, cudaStream_t s) {
  IndexBase* ix = sh->ix;
  const int W = sh->world, r = sh->rank;
  const int64_t nq = rd.nq;
  const int k = rd.k;
  const size_t qb = ix->query_row_bytes();
  if (L.last && L.last != s && L.done) B200VS_CUDA(cudaStreamWaitEvent(s, L.done, 0));
  SearchCtx sc = make_ctx(ix, rd.sp, s);
  const void* q = xq;
  int nprobe = 0;
  if (!sh->rows) {
    nprobe = ix->resolve_nprobe_api(sc);
    const int64_t per = (nq + W - 1) / W;
    // cosine: normalise once (NormalizeVectorForFaiss), the coarse pass and the list scan both take prepared queries
    if (!ix->binary()) q = ix->prepare_queries(nq, static_cast<const float*>(xq), s);
    // 1) coarse quantiser on this rank's slice, all-gather of the probe table (in place)
    L.probes.reserve((size_t)per * W * nprobe, 0, s);
    const int64_t q0 = std::min<int64_t>(nq, per * r), q1 = std::min<int64_t>(nq, per * (r + 1));
    long long* mine = L.probes.p + (size_t)per * r * nprobe;
    if (q1 - q0 < per) fill_ll_kernel<<<(unsigned)cdiv(per * nprobe, 256), 256, 0, s>>>(mine, per * nprobe, -1);
    if (q1 > q0) ix->coarse(q1 - q0, static_cast<const unsigned char*>(q) + (size_t)q0 * qb, true, nprobe, 0, ix->nlist_now(), nullptr, mine, s);
    ix->phase(IndexBase::PH_COMM, s);
    if (W > 1) B200VS_NCCL(nccl().AllGather(mine, L.probes.p, (size_t)per * nprobe, ncclInt64, L.comm, s));
    ix->phase(IndexBase::PH_OTHER, s);
  }
  // 2) scan of the probed lists this rank owns, or search of the rank's rows -> exact local results
  L.od.reserve((size_t)nq * k, 0, s);
  L.oi.reserve((size_t)nq * k, 0, s);
  const MergeKey key = merge_key(sh, rd.kind);
  SearchReq req;
  req.nq = nq; req.xq = q; req.k = k; req.sc = &sc; req.od = L.od.p; req.oi = L.oi.p;
  if (!sh->rows) { req.prepared = true; req.probes = L.probes.p; req.nprobe = nprobe; }
  req.raw = key.raw;
  req.deep = rd.kind == READ_DEEP;
  if (rd.kind == READ_RANGE) {
    req.range = true; req.radius = rd.radius;
    req.oc = ix->scratch.alloc<int>((size_t)nq);  // local counts: the merged rows are counted again by the finish
  }
  // a NaN radius admits no row (DESIGN.md 4.6): this rank contributes empty lists, and still joins the all-gather
  if (req.range && std::isnan(req.radius)) fill_empty(req, s);
  else ix->search(req, s);
  if (key.neg) launch_negate(L.od.p, nq * k, s);  // ip -> -ip
  // 3) the all-gather of the packed per-shard results + merge
  gather_merge(sh, L, nq, k, req.deep, out_dist, out_ids, s);
  if (!L.done) B200VS_CUDA(cudaEventCreateWithFlags(&L.done, cudaEventDisableTiming));
  B200VS_CUDA(cudaEventRecord(L.done, s));
  L.last = s;
  // 4) the finish: the merged key -> the API distance, the range counts
  if (key.neg || req.range) {
    merge_finish_kernel<<<(unsigned)cdiv(nq * k, 256), 256, 0, s>>>(out_dist, out_ids, nq, k, key.neg ? 1 : 0, out_counts);
    B200VS_CUDA(cudaGetLastError());
    ix->launch_count(1);
  }
  ix->phases_finish(s);
}

// Refusals of a sharded read decided from its arguments alone, so that every rank refuses alike; each kind keeps the order
// of its single-index call's refusals.  false: a top-k or deep read with k <= 0, OK with nothing to do.
bool check_read(const b200vs_shard* sh, const ShardRead& rd) {
  const IndexBase* ix = sh->ix;
  check_row_type(sh, rd.binary_call);
  if (rd.nq <= 0 || !rd.xq) fail(B200VS_EILLEGAL_PARAMETERS, "vector_with_ids is empty");
  if (rd.kind == READ_RANGE) {
    if (ix->type == B200VS_HNSW) fail(B200VS_EVECTOR_NOT_SUPPORT, "RangeSearch not support in Hnsw!!!");  // as b200vs_range_search
    if (rd.k <= 0 || rd.k > 4096) fail(B200VS_EILLEGAL_PARAMETERS, "max_results must be in [1, 4096]");
    if (!rd.od || !rd.oi || !rd.oc) fail(B200VS_EILLEGAL_PARAMETERS, "bad range-search outputs");
    if (ix->binary() && std::isnan(rd.radius)) fail(B200VS_EILLEGAL_PARAMETERS, "radius is NaN");  // as b200vs_range_search_binary
    return true;
  }
  if (rd.k <= 0) return false;
  if (rd.kind == READ_DEEP) {  // b200vs_search_deep's refusals, in its order
    if (rd.k > kDeepMaxK) fail(B200VS_EILLEGAL_PARAMETERS, "topk above " + std::to_string(kDeepMaxK));
    if (ix->type == B200VS_HNSW) fail(B200VS_EVECTOR_NOT_SUPPORT, "deep top-k is not implemented for HNSW");
  }
  if (!rd.od || !rd.oi) fail(B200VS_EILLEGAL_PARAMETERS, "null output");
  return true;
}

// The host-pointer reads: every rank passes the SAME batch; each rank uploads only its slice and the slices are all-gathered
// over NVLink, so the PCIe traffic per rank does not grow with the world size.  Returns the batch on the device.  Query rows
// are query_row_bytes() each (FP32, or packed bits on a binary index) and travel as bytes.
const void* upload_batch(b200vs_shard* sh, b200vs_shard::SLane& L, int64_t nq, const void* xq, cudaStream_t s) {
  const int W = sh->world, r = sh->rank;
  const size_t qb = sh->ix->query_row_bytes();
  const int64_t per = (nq + W - 1) / W;
  L.q_all.reserve((size_t)per * W * qb, 0, s);
  const int64_t q0 = std::min<int64_t>(nq, per * r), q1 = std::min<int64_t>(nq, per * (r + 1));
  unsigned char* mine = L.q_all.p + (size_t)per * r * qb;
  const unsigned char* src = static_cast<const unsigned char*>(xq);
  if (q1 > q0) B200VS_CUDA(cudaMemcpyAsync(mine, src + (size_t)q0 * qb, (size_t)(q1 - q0) * qb, cudaMemcpyHostToDevice, s));
  if (q1 - q0 < per) B200VS_CUDA(cudaMemsetAsync(mine + (size_t)(q1 - q0) * qb, 0, (size_t)(per - (q1 - q0)) * qb, s));
  if (W > 1) B200VS_NCCL(nccl().AllGather(mine, L.q_all.p, (size_t)per * qb, ncclUint8, L.comm, s));
  return L.q_all.p;
}

// The body of every sharded read entry point.  The turn of batch `seq` comes first, so that every call uses its sequence
// number exactly once, a refused one included; then check_read, the rw lock, the device and a lane on the read's stream,
// the refusals every rank meets alike before the first collective, and shard_stream (host pointers: the batch uploaded
// before it, the results copied back after it).  The lane is released before the host waits for a null-stream call, so the
// lane's next batch may be enqueued behind this one.
int shard_read(b200vs_shard* h, const ShardRead& rd) {
  return guarded([&]() -> int {
    b200vs_shard* sh = get(h);
    IndexBase* ix = sh->ix;
    cudaStream_t s;
    {
      SeqLane sl(sh, rd.seq);
      if (!check_read(sh, rd)) return B200VS_OK;
      std::shared_lock<std::shared_mutex> rl(ix->rw);
      ix->set_device();
      s = rd.stream ? (cudaStream_t)rd.stream : sl.lane->own;
      LaneGuard lane(ix, s);
      ix->check_probe_search(rd.nq, rd.k, rd.kind == READ_DEEP);
      if (sh->rows) ix->check_row_search(rd.k, rd.sp);
      ix->reset_stats();
      b200vs_shard::SLane& L = *sl.lane;
      if (rd.on_device) {
        shard_stream(sh, L, rd, rd.xq, rd.od, (long long*)rd.oi, rd.oc, s);
      } else {
        const size_t nk = (size_t)rd.nq * rd.k;
        const void* q = upload_batch(sh, L, rd.nq, rd.xq, s);
        float* dd = ix->scratch.alloc<float>(nk);
        long long* di = ix->scratch.alloc<long long>(nk);
        int* dc = rd.kind == READ_RANGE ? ix->scratch.alloc<int>((size_t)rd.nq) : nullptr;
        shard_stream(sh, L, rd, q, dd, di, dc, s);
        B200VS_CUDA(cudaMemcpyAsync(rd.od, dd, nk * 4, cudaMemcpyDeviceToHost, s));
        B200VS_CUDA(cudaMemcpyAsync(rd.oi, di, nk * 8, cudaMemcpyDeviceToHost, s));
        if (dc) B200VS_CUDA(cudaMemcpyAsync(rd.oc, dc, (size_t)rd.nq * 4, cudaMemcpyDeviceToHost, s));
      }
    }
    if (!rd.stream) B200VS_CUDA(cudaStreamSynchronize(s));
    return B200VS_OK;
  });
}

// Replicate rank `root`'s trained state on every rank (b200vs_shard_broadcast_state; the caller holds add_mu).  The length
// goes first, 0 when the root has no state, so that every rank refuses together.
void broadcast_state_locked(b200vs_shard* sh, int root) {
  IndexBase* ix = sh->ix;
  ix->set_device();
  const long long mine = sh->rank == root ? (long long)ix->get_state(nullptr, 0) : 0;
  const long long need = all_gather_host(sh, &mine)[root];
  if (need <= 0) fail(B200VS_EVECTOR_NOT_TRAIN, "root has no trained state");
  std::vector<unsigned char> blob;
  DevBuf<unsigned char> db;
  local_step(sh, true, "shard broadcast_state", [&] {
    blob.resize((size_t)need);
    if (sh->rank == root) ix->get_state(blob.data(), blob.size());
    db.reserve((size_t)need, 0, sh->ws);
    if (sh->rank == root) B200VS_CUDA(cudaMemcpyAsync(db.p, blob.data(), (size_t)need, cudaMemcpyHostToDevice, sh->ws));
  });
  if (sh->world > 1) B200VS_NCCL(nccl().Broadcast(db.p, db.p, (size_t)need, ncclUint8, root, sh->lanes[0]->comm, sh->ws));
  // the install is agreed too: every rank returns the same status, and the caller's next collective finds every rank
  local_step(sh, true, "shard broadcast_state", [&] {
    if (sh->rank != root) {
      B200VS_CUDA(cudaMemcpyAsync(blob.data(), db.p, (size_t)need, cudaMemcpyDeviceToHost, sh->ws));
      B200VS_CUDA(cudaStreamSynchronize(sh->ws));
      ix->set_state(blob.data(), blob.size());
    } else {
      B200VS_CUDA(cudaStreamSynchronize(sh->ws));
    }
  });
}

// b200vs_shard_train on IVF_FLAT and IVF_PQ, b200vs_shard_train_binary on BINARY_IVF_FLAT (x: packed rows).  The per-rank row
// counts are exchanged first, so that a refusal for too few rows happens on every rank at once.  Coarse stage: each rank
// clusters its rows into nlist / world centroids with the k-means of its type's own train, and every rank's status is
// agreed before the one all-gather.  IVF_FLAT and BINARY_IVF_FLAT: every rank installs the gathered centroids.  IVF_PQ:
// rank 0 trains the codebooks with train's PQ rule on the residuals of its rows to the global centroids, and the state
// broadcast replicates the result.  At world = 1 this is b200vs_train[_binary] step for step, so the trained state is
// byte-equal.  on_device (b200vs_shard_rebuild_from; IVF_FLAT and BINARY_IVF_FLAT): x is on the index's device, prepared
// FP32 rows or padded binary rows [n, ceil(dim / 32)] words, and is clustered as b200vs_rebuild_from clusters its rows.
void shard_train_locked(b200vs_shard* sh, int64_t n, const void* xv, bool on_device) {
  IndexBase* ix = sh->ix;
  const bool pq = ix->type == B200VS_IVF_PQ;
  const int W = sh->world, nlist = ix->params.nlist > 0 ? ix->params.nlist : 2048;
  if (nlist % W != 0) fail(B200VS_EILLEGAL_PARAMETERS, "shard_train: nlist must be a multiple of the world size");
  if (pq && ix->sub_type() == B200VS_FLAT) fail(B200VS_EVECTOR_NOT_SUPPORT, "an IVF_PQ index in inner-Flat mode has no inverted lists to shard");
  const int nl = nlist / W;
  ix->set_device();
  const long long rows = xv ? (long long)n : 0;  // a null x counts as none
  const std::vector<long long> counts = all_gather_host(sh, &rows);
  for (int r = 0; r < W; ++r)
    if (counts[r] < nl)
      fail(B200VS_EILLEGAL_PARAMETERS, "shard_train: rank " + std::to_string(r) + " has fewer training rows than nlist / world centroids");
  if (pq && counts[0] < 256LL * ivf_pq_ksub(ix))
    fail(B200VS_EILLEGAL_PARAMETERS, "shard_train: rank 0 needs 256 * 2^nbits training rows for the PQ codebooks");
  int64_t total = 0;
  for (const long long c : counts) total += c;
  std::vector<unsigned char> blob;
  if (ix->binary()) {
    std::vector<uint8_t> local;
    const uint8_t* x = on_device ? nullptr : static_cast<const uint8_t*>(xv);
    const uint32_t* words = on_device ? static_cast<const uint32_t*>(xv) : nullptr;
    check(agree(sh, attempt([&] { binary_ivf_train_coarse(ix, n, x, words, nl, local); }), "shard train"));
    binary_ivf_train_state(ix, all_gather_host(sh, local.data(), local.size()), blob);
    local_step(sh, true, "shard train", [&] { ix->set_state(blob.data(), blob.size()); });
    sh->train_rows_set = total;
    return;
  }
  const float* x = static_cast<const float*>(xv);
  std::vector<float> local;
  check(agree(sh, attempt([&] {
    if (pq) ivf_pq_train_coarse(ix, n, x, nl, local);
    else ivf_flat_train_coarse(ix, n, x, on_device, nl, local);
  }), "shard train"));
  const std::vector<float> cent = all_gather_host(sh, local.data(), local.size());
  if (!pq) {
    ivf_flat_train_state(ix, cent, blob);
    local_step(sh, true, "shard train", [&] { ix->set_state(blob.data(), blob.size()); });
    sh->train_rows_set = total;
    return;
  }
  local_step(sh, true, "shard train", [&] {
    if (sh->rank != 0) return;
    ivf_pq_train_state(ix, n, x, cent, blob);
    ix->set_state(blob.data(), blob.size());
  });
  broadcast_state_locked(sh, 0);
  sh->train_rows_set = total;
}

// Every rank's live rows, summed (collective): the training size the set's rule takes after a state broadcast or a load, as
// b200vs_set_trained_state and b200vs_load take the live count of one index
int64_t live_rows_set(b200vs_shard* sh) {
  long long mine = 0;
  {
    std::shared_lock<std::shared_mutex> rl(sh->ix->rw);
    mine = (long long)sh->ix->count();
  }
  int64_t sum = 0;
  for (const long long v : all_gather_host(sh, &mine)) sum += v;
  return sum;
}

// b200vs_shard_create (float indexes) and b200vs_shard_create_binary (binary ones)
int shard_create(b200vs_index* idx, int32_t rank, int32_t world, const uint8_t* id, int32_t lanes, b200vs_shard** out, bool binary_call) {
  return guarded([&]() -> int {
    if (!out) fail(B200VS_EILLEGAL_PARAMETERS, "out is null");
    *out = nullptr;
    IndexBase* ix = index_impl(idx);
    if (binary_call && !ix->binary()) fail(B200VS_EILLEGAL_PARAMETERS, "binary entry point on a float index");
    if (!binary_call && ix->binary())
      fail(B200VS_EVECTOR_NOT_SUPPORT, "sharding is implemented for FLAT and HNSW (by rows), IVF_FLAT and IVF_PQ (by list); binary indexes "
                                       "shard through b200vs_shard_create_binary");
    const bool rows = shard_by_rows(ix->type);  // else shard_by_lists
    if (ix->type == B200VS_IVF_PQ && ix->sub_type() == B200VS_FLAT)
      fail(B200VS_EVECTOR_NOT_SUPPORT, "an IVF_PQ index in inner-Flat mode (too few training rows) has no inverted lists to shard");
    if (rows && ix->count() + ix->deleted_count() > 0)
      fail(B200VS_EVECTOR_NOT_SUPPORT, "a row-sharded index must be empty when its shard is created");
    if (world < 1 || rank < 0 || rank >= world) fail(B200VS_EILLEGAL_PARAMETERS, "bad rank / world");
    if (world > ROUTE_MAX_WORLD) fail(B200VS_EILLEGAL_PARAMETERS, "sharding supports at most 1024 ranks");
    if (world > 1 && !id) fail(B200VS_EILLEGAL_PARAMETERS, "null communicator id");
    lanes = std::max(1, std::min(lanes <= 0 ? 2 : lanes, kLanes));
    std::unique_ptr<b200vs_shard> sh(new b200vs_shard());
    sh->ix = ix; sh->rank = rank; sh->world = world; sh->nlanes = lanes; sh->rows = rows;
    ix->set_device();
    B200VS_CUDA(cudaStreamCreateWithFlags(&sh->ws, cudaStreamNonBlocking));
    for (int c = 0; c < lanes; ++c) {
      sh->lanes.emplace_back(new b200vs_shard::SLane());
      B200VS_CUDA(cudaStreamCreateWithFlags(&sh->lanes.back()->own, cudaStreamNonBlocking));
    }
    if (world > 1) {
      ncclUniqueId u;
      memcpy(&u, id, sizeof(u));
      B200VS_NCCL(nccl().CommInitRank(&sh->lanes[0]->comm, world, u, rank));
      for (int c = 1; c < lanes; ++c) B200VS_NCCL(nccl().CommSplit(sh->lanes[0]->comm, 0, rank, &sh->lanes[c]->comm, nullptr));
    }
    *out = sh.release();
    return B200VS_OK;
  });
}

// Distributed training: every rank clusters ITS training rows into nlist / world centroids (faiss::Clustering shape, as
// b200vs_train), the blocks are all-gathered into the replicated global table.  Build time stays flat as ranks are added.
int shard_train(b200vs_shard* h, int64_t n, const void* x, bool binary_call) {
  return guarded([&]() -> int {
    b200vs_shard* sh = get(h);
    check_row_type(sh, binary_call);
    if (sh->rows) return B200VS_OK;  // FLAT, BINARY_FLAT and HNSW have nothing to train (b200vs_train is a no-op on them too)
    std::lock_guard<Gate> g(sh->add_mu);
    shard_train_locked(sh, n, x, false);
    return B200VS_OK;
  });
}

}  // namespace

extern "C" {

int b200vs_shard_unique_id(uint8_t id[B200VS_SHARD_ID_BYTES]) {
  return guarded([&]() -> int {
    if (!id) fail(B200VS_EILLEGAL_PARAMETERS, "null id");
    static_assert(sizeof(ncclUniqueId) <= B200VS_SHARD_ID_BYTES, "ncclUniqueId must fit the ABI's id blob");
    ncclUniqueId u;
    B200VS_NCCL(nccl().GetUniqueId(&u));
    memset(id, 0, B200VS_SHARD_ID_BYTES);
    memcpy(id, &u, sizeof(u));
    return B200VS_OK;
  });
}

int b200vs_shard_create(b200vs_index* idx, int32_t rank, int32_t world, const uint8_t id[B200VS_SHARD_ID_BYTES], int32_t lanes, b200vs_shard** out) {
  return shard_create(idx, rank, world, id, lanes, out, false);
}

int b200vs_shard_create_binary(b200vs_index* idx, int32_t rank, int32_t world, const uint8_t id[B200VS_SHARD_ID_BYTES], int32_t lanes,
                               b200vs_shard** out) {
  return shard_create(idx, rank, world, id, lanes, out, true);
}

void b200vs_shard_destroy(b200vs_shard* sh) {
  try { delete sh; } catch (...) {}
}

int b200vs_shard_list_range(b200vs_shard* h, int32_t rank, int32_t* begin, int32_t* end) {
  return guarded([&]() -> int {
    b200vs_shard* sh = get(h);
    if (sh->rows) fail(B200VS_EVECTOR_NOT_SUPPORT, "a row-sharded index has no inverted lists");
    if (rank < 0 || rank >= sh->world) fail(B200VS_EILLEGAL_PARAMETERS, "bad rank");
    const int nl = sh->ix->nlist_now(), per = sh->lists_per_rank();
    if (begin) *begin = std::min(nl, per * rank);
    if (end) *end = std::min(nl, per * (rank + 1));
    return B200VS_OK;
  });
}

int b200vs_shard_train(b200vs_shard* h, int64_t n, const float* x) { return shard_train(h, n, x, false); }
int b200vs_shard_train_binary(b200vs_shard* h, int64_t n, const uint8_t* x) { return shard_train(h, n, x, true); }

// Replicate rank `root`'s trained state (centroids; IVF-PQ: and codebooks) on every rank.
int b200vs_shard_broadcast_state(b200vs_shard* h, int32_t root) {
  return guarded([&]() -> int {
    b200vs_shard* sh = get(h);
    // an HNSW state blob is a whole graph: replicating it would put every row on every rank
    if (sh->rows) fail(B200VS_EVECTOR_NOT_SUPPORT, "a row-sharded index has no replicated trained state");
    if (root < 0 || root >= sh->world) fail(B200VS_EILLEGAL_PARAMETERS, "bad root");
    std::lock_guard<Gate> g(sh->add_mu);
    broadcast_state_locked(sh, root);
    sh->train_rows_set = live_rows_set(sh);
    return B200VS_OK;
  });
}

}  // extern "C"

namespace {

// assignment of n device rows (raw, in the index's row format) -> prepared rows (cosine: normalised copy) + lists, on the
// write stream.  Returns the prepared rows (either x itself or `prep`).
const void* assign_rows(b200vs_shard* sh, int64_t n, const void* x_dev, DevBuf<float>& prep, DevBuf<long long>& lists) {
  IndexBase* ix = sh->ix;
  cudaStream_t s = sh->ws;
  const void* xp = x_dev;
  if (ix->metric == B200VS_COSINE) {
    prep.reserve((size_t)n * ix->dim, 0, s);
    B200VS_CUDA(cudaMemcpyAsync(prep.p, x_dev, (size_t)n * ix->dim * 4, cudaMemcpyDeviceToDevice, s));
    launch_normalize_faiss(prep.p, n, ix->dim, s);
    xp = prep.p;
  }
  lists.reserve((size_t)n, 0, s);
  {
    std::shared_lock<std::shared_mutex> rl(ix->rw);
    LaneGuard lane(ix, s);
    ix->assign_lists_dev(n, xp, lists.p, s);
  }
  return xp;
}

// Moves n device rows (rows of rb bytes, ids and, list-sharded, lists) to their owners: a stable partition by owner on the
// device (route_*_kernel), the counts-matrix all-gather, and one grouped ncclSend / ncclRecv.  A rank receives rank 0's
// rows first, then rank 1's, ..., each in its caller's order; at world 1 the partitioned rows are the received ones.
struct Routed {
  DevBuf<unsigned char> x;
  DevBuf<long long> ids, lists;
  long long n = 0;
};
// agreed (b200vs_shard_rebuild_from): the partition (the send copy) and the reservation of the received copy are local_steps
// with a status agreement each, so a rank that cannot hold them fails on every rank before the exchange.
template <class Owner>
void route_rows(b200vs_shard* sh, int64_t n, const void* xv, int rb, const long long* ids, const long long* lists, Owner owner, Routed& out,
                bool agreed = false) {
  const int W = sh->world, r = sh->rank, d = rb;  // d: bytes per row below
  const unsigned char* x = static_cast<const unsigned char*>(xv);
  cudaStream_t s = sh->ws;
  ncclComm_t comm = sh->lanes[0]->comm;
  Routed snd;
  DevBuf<long long> cnt_all, tile_off;
  DevBuf<int> tile_cnt;
  long long* mine = nullptr;
  // stable partition by owner on the device; this rank's row of the counts matrix
  local_step(sh, agreed, "shard routing", [&] {
  cnt_all.reserve((size_t)W * W, 0, s);
  mine = cnt_all.p + (size_t)r * W;
  if (n) {
    const long long ntiles = cdiv(n, ROUTE_THREADS);
    const size_t smem = (size_t)ROUTE_WARPS * W * 4;
    tile_cnt.reserve((size_t)ntiles * W, 0, s); tile_off.reserve((size_t)ntiles * W, 0, s);
    snd.x.reserve((size_t)n * d, 0, s); snd.ids.reserve((size_t)n, 0, s);
    if (Owner::kLists) snd.lists.reserve((size_t)n, 0, s);
    route_count_kernel<<<(unsigned)ntiles, ROUTE_THREADS, smem, s>>>(Owner::kLists ? lists : ids, n, W, owner, tile_cnt.p);
    route_offsets_kernel<<<1, ROUTE_SCAN_THREADS, 0, s>>>(tile_cnt.p, ntiles, W, tile_off.p, mine);
    route_scatter_kernel<<<(unsigned)ntiles, ROUTE_THREADS, smem, s>>>(x, ids, lists, n, d, W, owner, tile_off.p, snd.x.p, snd.ids.p,
                                                                       snd.lists.p);
    B200VS_CUDA(cudaGetLastError());
  } else {
    B200VS_CUDA(cudaMemsetAsync(mine, 0, (size_t)W * 8, s));
  }
  });
  // counts matrix: every rank learns how many rows each peer sends it
  if (W > 1) B200VS_NCCL(nccl().AllGather(mine, cnt_all.p, (size_t)W, ncclInt64, comm, s));
  std::vector<long long> h_cnt((size_t)W * W);
  B200VS_CUDA(cudaMemcpyAsync(h_cnt.data(), cnt_all.p, (size_t)W * W * 8, cudaMemcpyDeviceToHost, s));
  B200VS_CUDA(cudaStreamSynchronize(s));
  std::vector<long long> send_off(W + 1, 0), recv_off(W + 1, 0);
  for (int w = 0; w < W; ++w) {
    send_off[w + 1] = send_off[w] + h_cnt[(size_t)r * W + w];
    recv_off[w + 1] = recv_off[w] + h_cnt[(size_t)w * W + r];
  }
  out.n = recv_off[W];
  if (W == 1) {  // a world of one receives exactly what it sends
    out.x.swap(snd.x); out.ids.swap(snd.ids); out.lists.swap(snd.lists);
    return;
  }
  const size_t cap = (size_t)std::max<long long>(out.n, 1);
  local_step(sh, agreed, "shard routing", [&] {
    out.x.reserve(cap * d, 0, s); out.ids.reserve(cap, 0, s);
    if (Owner::kLists) out.lists.reserve(cap, 0, s);
  });
  B200VS_NCCL(nccl().GroupStart());
  for (int w = 0; w < W; ++w) {
    const long long so = send_off[w], sc = send_off[w + 1] - so, ro = recv_off[w], rc = recv_off[w + 1] - ro;
    if (sc) {
      B200VS_NCCL(nccl().Send(snd.x.p + (size_t)so * d, (size_t)sc * d, ncclUint8, w, comm, s));
      B200VS_NCCL(nccl().Send(snd.ids.p + so, (size_t)sc, ncclInt64, w, comm, s));
      if (Owner::kLists) B200VS_NCCL(nccl().Send(snd.lists.p + so, (size_t)sc, ncclInt64, w, comm, s));
    }
    if (rc) {
      B200VS_NCCL(nccl().Recv(out.x.p + (size_t)ro * d, (size_t)rc * d, ncclUint8, w, comm, s));
      B200VS_NCCL(nccl().Recv(out.ids.p + ro, (size_t)rc, ncclInt64, w, comm, s));
      if (Owner::kLists) B200VS_NCCL(nccl().Recv(out.lists.p + ro, (size_t)rc, ncclInt64, w, comm, s));
    }
  }
  B200VS_NCCL(nccl().GroupEnd());
}

// The collective add of both shard kinds.  List-sharded (IVF_FLAT, IVF_PQ): the sender assigns each row to its list, and the
// row travels PREPARED (normalised for cosine) with its list to the list's owner, which appends it there.  Row-sharded
// (FLAT, HNSW): every row travels RAW to owner(id) (Flat and HNSW normalise cosine rows differently, so the owner's add
// normalises), and the owner runs the single-index add on the rows it received, in arrival order (an HNSW graph depends on
// it).  Either way the owner makes one add of the device rows it received.  Before any rank changes anything, every owner
// checks that add (check_add: a negative id for every type, a repeated id for FLAT, max_elements for HNSW) and the statuses
// are all-gathered: every rank returns the first refusal in rank order, or adds.  batched: b200vs_hnsw_add_batched with
// `batch`.  Rows are in the index's row format (FP32, or packed bits on the binary types, which travel as they are: a
// binary row has no normalisation).  agreed (b200vs_shard_rebuild_from): every local step before a collective (the
// assignment and its cosine copy, the routing's copies) and the final add are agreed, so a device failure on one rank is
// returned by every rank.
void shard_add_impl(b200vs_shard* sh, int64_t n, const void* x_dev, const long long* ids_dev, bool batched, int batch, bool agreed = false) {
  IndexBase* ix = sh->ix;
  const int rb = (int)ix->query_row_bytes();
  cudaStream_t s = sh->ws;
  ix->set_device();
  Routed rv;
  if (sh->rows) {
    route_rows(sh, n, x_dev, rb, ids_dev, nullptr, RowOwner{}, rv, agreed);
  } else {
    DevBuf<float> prep;
    DevBuf<long long> lists;
    const void* xp = x_dev;
    local_step(sh, agreed, "shard add", [&] { if (n > 0) xp = assign_rows(sh, n, x_dev, prep, lists); });
    route_rows(sh, n, xp, rb, ids_dev, lists.p, ListOwner{sh->lists_per_rank()}, rv, agreed);
  }
  std::vector<int64_t> hid((size_t)rv.n);  // the host ids check_add and the add take
  local_step(sh, agreed, "shard add", [&] {
    if (!hid.empty()) B200VS_CUDA(cudaMemcpyAsync(hid.data(), rv.ids.p, hid.size() * 8, cudaMemcpyDeviceToHost, s));
    B200VS_CUDA(cudaStreamSynchronize(s));
  });
  AddReq req = AddReq::device(rv.n, rv.x.p, rv.ids.p, rv.lists.p, false, sh->rows ? AddReq::RAW : AddReq::PREPARED);
  req.ids = hid.data();
  req.batched = batched;
  req.batch = batch;
  // status agreement
  check(agree(sh, attempt([&] { ix->check_add(req); }), "shard add"));
  local_step(sh, agreed, "shard add", [&] { if (rv.n) ix->add(req); });
}

// upload of host rows (query_row_bytes() each) to the write stream, for the host-pointer variants of the collective adds
void upload_rows(b200vs_shard* sh, int64_t n, const void* x, const int64_t* ids, DevBuf<unsigned char>& dx, DevBuf<long long>& di) {
  if (!n) return;
  const size_t rb = sh->ix->query_row_bytes();
  dx.reserve((size_t)n * rb, 0, sh->ws); di.reserve((size_t)n, 0, sh->ws);
  B200VS_CUDA(cudaMemcpyAsync(dx.p, x, (size_t)n * rb, cudaMemcpyHostToDevice, sh->ws));
  B200VS_CUDA(cudaMemcpyAsync(di.p, ids, (size_t)n * 8, cudaMemcpyHostToDevice, sh->ws));
  B200VS_CUDA(cudaStreamSynchronize(sh->ws));
}

// Rows per list of the whole sharded index: every rank's counts counts_dev[nlist] summed over the ranks (collective).
std::vector<int64_t> sum_list_counts(b200vs_shard* sh, unsigned long long* counts_dev, int nlist) {
  if (sh->world > 1) B200VS_NCCL(nccl().AllReduce(counts_dev, counts_dev, (size_t)nlist, ncclUint64, ncclSum, sh->lanes[0]->comm, sh->ws));
  std::vector<int64_t> cnt((size_t)nlist);
  B200VS_CUDA(cudaMemcpyAsync(cnt.data(), counts_dev, (size_t)nlist * 8, cudaMemcpyDeviceToHost, sh->ws));
  B200VS_CUDA(cudaStreamSynchronize(sh->ws));
  return cnt;
}

// Pre-sizes the lists this rank owns from the index-wide counts in one arena allocation; the others stay empty here.
void reserve_owned_lists(b200vs_shard* sh, std::vector<int64_t>& cnt) {
  const int nlist = (int)cnt.size(), per = sh->lists_per_rank();
  for (int l = 0; l < nlist; ++l)
    if (std::min(sh->world - 1, l / per) != sh->rank) cnt[l] = 0;  // lists owned elsewhere stay empty here
  sh->ix->reserve_lists(cnt.data(), nlist);
}

// ---------------------------------------------------------------------------------------------
// Snapshots (b200vs_shard_save / b200vs_shard_load)
// ---------------------------------------------------------------------------------------------
// A snapshot of W ranks is <prefix>.<r>-of-<W> per rank, each in its index's own Save container, and <prefix>.manifest:
// ManifestHdr, then one RankEntry per rank.
struct ManifestHdr {
  char magic[8];
  int32_t version, type, metric, dim;
  int32_t nlist, pq_m, pq_nbits, hnsw_m, hnsw_efc, world;  // the creation parameters that decide results (0: not used by the type)
  int64_t max_elements;
  int64_t state_len;      // list-sharded: bytes of the replicated trained state, 0 when untrained
  uint64_t state_digest;  // and its digest
};
static_assert(sizeof(ManifestHdr) == 72, "manifest header layout");
struct RankEntry {
  int64_t rows, bytes;  // live rows of the rank, size of its file
  uint64_t digest;      // of the whole file
};
constexpr char kManifestMagic[8] = {'B', '2', 'V', 'S', 'S', 'H', 'M', '1'};
constexpr int32_t kManifestVersion = 1;
constexpr size_t kRestoreChunkBytes = 64u << 20;  // rows read, uploaded and routed per restore round

// 64-bit content digest of a byte stream, fed in pieces of any size: 32-byte blocks, word j of a block through a
// multiply-rotate mix into lane j (four independent chains, so the host digests at memory speed), the zero-padded tail
// and the length last, the lanes folded with splitmix64's finalizer.  A check against corrupt, truncated or swapped
// files, not a cryptographic hash.
struct Digest {
  uint64_t h[4] = {0x243f6a8885a308d3ULL, 0x13198a2e03707344ULL, 0xa4093822299f31d0ULL, 0x082efa98ec4e6c89ULL};
  uint64_t len = 0;
  unsigned char tail[32];
  size_t nt = 0;
  static uint64_t mix(uint64_t h, uint64_t w) {
    h ^= w * 0x9e3779b97f4a7c15ULL;
    return ((h << 31) | (h >> 33)) * 0xbf58476d1ce4e5b9ULL;
  }
  void block(const unsigned char* b) {
    uint64_t w[4];
    memcpy(w, b, 32);
    for (int j = 0; j < 4; ++j) h[j] = mix(h[j], w[j]);
  }
  void update(const void* p, size_t n) {
    const unsigned char* b = static_cast<const unsigned char*>(p);
    len += n;
    if (nt) {
      const size_t m = std::min(n, 32 - nt);
      memcpy(tail + nt, b, m);
      nt += m; b += m; n -= m;
      if (nt < 32) return;
      block(tail);
      nt = 0;
    }
    for (; n >= 32; n -= 32, b += 32) block(b);
    memcpy(tail, b, n);
    nt = n;
  }
  uint64_t value() const {
    Digest c = *this;
    if (c.nt) {
      memset(c.tail + c.nt, 0, 32 - c.nt);
      c.block(c.tail);
    }
    uint64_t z = c.len;
    for (int j = 0; j < 4; ++j) {
      z = mix(z, c.h[j]);
      z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
      z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
      z ^= z >> 31;
    }
    return z;
  }
};

struct File {
  FILE* f = nullptr;
  File(const std::string& path, const char* mode) : f(fopen(path.c_str(), mode)) {
    if (!f) fail(B200VS_EINTERNAL, "cannot open " + path);
  }
  ~File() { if (f) fclose(f); }
  File(const File&) = delete;
  File& operator=(const File&) = delete;
  int64_t size() {
    fseeko(f, 0, SEEK_END);
    const int64_t n = ftello(f);
    fseeko(f, 0, SEEK_SET);
    return n;
  }
  void read(void* p, size_t n) {
    if (n && fread(p, 1, n, f) != n) fail(B200VS_EINTERNAL, "short read / truncated snapshot file");
  }
  void write(const void* p, size_t n) {
    if (n && fwrite(p, 1, n, f) != n) fail(B200VS_EINTERNAL, "short write");
  }
  void close() {
    FILE* g = f;
    f = nullptr;
    if (fclose(g) != 0) fail(B200VS_EINTERNAL, "short write");
  }
};

std::string rank_path(const std::string& prefix, int r, int W) {
  return prefix + "." + std::to_string(r) + "-of-" + std::to_string(W);
}

// The manifest header a snapshot of this index over W ranks carries (state fields left 0)
ManifestHdr manifest_of(const IndexBase* ix, int W) {
  ManifestHdr m;
  memset(&m, 0, sizeof(m));
  memcpy(m.magic, kManifestMagic, 8);
  m.version = kManifestVersion;
  m.type = ix->type; m.metric = ix->metric; m.dim = ix->dim; m.world = W;
  const b200vs_params& p = ix->params;
  if (shard_by_lists(ix->type)) m.nlist = p.nlist > 0 ? p.nlist : 2048;
  if (ix->type == B200VS_IVF_PQ) { m.pq_m = p.pq_m > 0 ? p.pq_m : 64; m.pq_nbits = p.pq_nbits > 0 ? p.pq_nbits : 8; }
  if (ix->type == B200VS_HNSW) { m.hnsw_m = p.hnsw_m; m.hnsw_efc = p.hnsw_efc; m.max_elements = p.max_elements; }
  return m;
}

// The trained state of a list-sharded index (empty when untrained)
std::vector<unsigned char> state_of(IndexBase* ix) {
  std::vector<unsigned char> blob((size_t)std::max<int64_t>(ix->get_state(nullptr, 0), 0));
  if (!blob.empty()) ix->get_state(blob.data(), blob.size());
  return blob;
}
uint64_t digest_of(const std::vector<unsigned char>& v) {
  Digest d;
  d.update(v.data(), v.size());
  return d.value();
}

// The index's writer lock held across a local snapshot step: adds wait, searches in flight finish first, and the step's own
// reader holds (RwSharedGuard) see this hold and do not lock again.
struct WriterHold {
  std::unique_lock<std::shared_mutex> lk;
  const IndexBase* prev;
  explicit WriterHold(IndexBase* ix) : lk(ix->rw), prev(RwSharedGuard::tl_held) { RwSharedGuard::tl_held = ix; }
  ~WriterHold() { RwSharedGuard::tl_held = prev; }
};

void shard_save_locked(b200vs_shard* sh, const std::string& prefix) {
  IndexBase* ix = sh->ix;
  const int r = sh->rank, W = sh->world;
  ix->set_device();
  const std::string mine = rank_path(prefix, r, W), tmp = mine + ".tmp", man = prefix + ".manifest", man_tmp = man + ".tmp";
  ManifestHdr mh = manifest_of(ix, W);
  RankEntry e{0, 0, 0};
  auto cleanup = [&] {  // temporary files only: an earlier snapshot under the same prefix stays as it was
    unlink(tmp.c_str());
    if (r == 0) unlink(man_tmp.c_str());
  };
  // 1) every rank writes its file under a temporary name
  Status st = agree(sh, attempt([&] {
    WriterHold hold(ix);
    ix->save(tmp);
    e.rows = ix->count();
    if (!sh->rows) {
      const std::vector<unsigned char> blob = state_of(ix);
      mh.state_len = (int64_t)blob.size();
      mh.state_digest = digest_of(blob);
    }
    File f(tmp, "rb");
    e.bytes = f.size();
    std::vector<unsigned char> buf(std::min<size_t>(kRestoreChunkBytes, (size_t)std::max<int64_t>(e.bytes, 1)));
    Digest d;
    for (int64_t at = 0; at < e.bytes; at += (int64_t)buf.size()) {
      const size_t m = (size_t)std::min<int64_t>((int64_t)buf.size(), e.bytes - at);
      f.read(buf.data(), m);
      d.update(buf.data(), m);
    }
    e.digest = d.value();
  }), "shard save");
  if (st.code != B200VS_OK) { cleanup(); check(st); }
  // 2) rank 0 writes the manifest under a temporary name
  const std::vector<RankEntry> ents = all_gather_host(sh, &e);
  st = agree(sh, attempt([&] {
    if (r != 0) return;
    File f(man_tmp, "wb");
    f.write(&mh, sizeof(mh));
    f.write(ents.data(), ents.size() * sizeof(RankEntry));
    f.close();
  }), "shard save");
  if (st.code != B200VS_OK) { cleanup(); check(st); }
  // 3) every file is renamed into place, the manifest last
  st = agree(sh, attempt([&] {
    if (rename(tmp.c_str(), mine.c_str()) != 0) fail(B200VS_EINTERNAL, "cannot rename " + tmp + " to " + mine);
  }), "shard save");
  if (st.code != B200VS_OK) { cleanup(); check(st); }
  check(agree(sh, attempt([&] {
    if (r == 0 && rename(man_tmp.c_str(), man.c_str()) != 0) fail(B200VS_EINTERNAL, "cannot rename " + man_tmp + " to " + man);
  }), "shard save"));
}

// One rank file of a snapshot, checked against its manifest entry: the sections before the rows are kept, the rows are
// read again by the restore rounds.
struct RankFile {
  std::string path;
  int64_t rows = 0, rows_at = 0;  // rows stored, and the file offset of the row section
  int rb = 0;                     // bytes per stored row: FP32 row, packed binary row or IVF-PQ code row
  std::vector<unsigned char> state;
  std::vector<int64_t> off, ids;  // list offsets [nlist + 1], ids [rows]
  int nlist() const { return (int)off.size() - 1; }
};

// bytes of one stored row of a rank file: an FP32 row, a packed binary row of dim / 8 bytes, or an IVF-PQ code row of
// ceil(M * nbits / 8) bytes
int restore_row_bytes(const IndexBase* ix, const ManifestHdr& mh) {
  return ix->type == B200VS_IVF_PQ ? (mh.pq_m * mh.pq_nbits + 7) / 8 : (int)ix->query_row_bytes();
}

// Reads and checks one rank file.  full = false: the header and the trained state only, for a rank that reads no file of
// its own but needs the state.  The header's sizes are checked against the file before anything is allocated from them.
RankFile read_rank_file(IndexBase* ix, const std::string& path, const RankEntry& ent, const ManifestHdr& mh, bool full) {
  RankFile rf;
  rf.path = path;
  File f(path, "rb");
  const int64_t fsize = f.size();
  if (full && fsize != ent.bytes) fail(B200VS_EINTERNAL, path + ": size differs from the manifest (truncated or replaced file)");
  Digest dg;
  auto rd = [&](void* p, size_t n) { f.read(p, n); dg.update(p, n); };
  int64_t state_len = 0, nlist = 0, count = 0, here = 0;
  bool lists = true;  // the file has a list-offset section
  const char* bad = "does not match the index (type / metric / dimension / nsubvector)";
  if (ix->type == B200VS_IVF_PQ) {  // "B2VSPQ01": int64 {magic, mode (0 untrained, 2 IVF-PQ), metric, dim, nlist, M, rows, state_len}
    int64_t h[8];
    rd(h, sizeof(h));
    here = sizeof(h);
    if (memcmp(h, "B2VSPQ01", 8) != 0 || h[2] != ix->metric || h[3] != ix->dim || h[5] != mh.pq_m) fail(B200VS_EINTERNAL, path + ": " + bad);
    if (h[1] == 2) { nlist = h[4]; count = h[6]; state_len = h[7]; }
    else if (h[1] == 0) lists = false;  // untrained: the header alone
    else fail(B200VS_EINTERNAL, path + ": an IVF_PQ index in inner-Flat mode is not a list-sharded snapshot");
  } else {
    IndexFileHdr h;
    rd(&h, sizeof(h));
    here = sizeof(h);
    if (memcmp(h.magic, ix->binary() ? "B2VSBIN1" : "B2VSIDX1", 8) != 0 || h.type != ix->type || h.metric != ix->metric || h.dim != ix->dim)
      fail(B200VS_EINTERNAL, path + ": " + bad);
    nlist = h.nlist; count = h.count; state_len = h.state_len;
  }
  rf.rb = restore_row_bytes(ix, mh);
  const double need = (double)state_len + (lists ? ((double)nlist + 1) * 8 : 0) + (double)count * (8 + (double)rf.rb);
  if (state_len < 0 || count < 0 || nlist < 0 || nlist > (1 << 24) || (lists && nlist < 1) || need > (double)(fsize - here) ||
      (full && need != (double)(fsize - here)))
    fail(B200VS_EINTERNAL, path + ": corrupt snapshot file (header sizes do not match the file)");
  rf.state.resize((size_t)state_len);
  rd(rf.state.data(), rf.state.size());
  if (shard_by_lists(ix->type) && ((int64_t)rf.state.size() != mh.state_len || digest_of(rf.state) != mh.state_digest))
    fail(B200VS_EINTERNAL, path + ": trained state differs from the manifest's");
  if (!full) return rf;
  if (lists) {
    rf.off.resize((size_t)nlist + 1);
    rd(rf.off.data(), rf.off.size() * 8);
  } else {
    rf.off.assign(2, 0);
  }
  rf.ids.resize((size_t)count);
  rd(rf.ids.data(), rf.ids.size() * 8);
  rf.rows = count;
  rf.rows_at = ftello(f.f);
  std::vector<unsigned char> buf(std::min<size_t>(kRestoreChunkBytes, (size_t)std::max<int64_t>(count * rf.rb, 1)));
  for (int64_t at = 0, total = count * rf.rb; at < total; at += (int64_t)buf.size()) {
    const size_t m = (size_t)std::min<int64_t>((int64_t)buf.size(), total - at);
    rd(buf.data(), m);
  }
  if (dg.value() != ent.digest) fail(B200VS_EINTERNAL, path + ": content differs from the manifest (swapped or replaced file)");
  if (ix->type != B200VS_HNSW && count != ent.rows) fail(B200VS_EINTERNAL, path + ": row count differs from the manifest");
  if (rf.off[0] != 0 || rf.off.back() != count) fail(B200VS_EINTERNAL, path + ": corrupt list offsets");
  for (size_t l = 0; l + 1 < rf.off.size(); ++l)
    if (rf.off[l] > rf.off[l + 1]) fail(B200VS_EINTERNAL, path + ": corrupt list offsets");
  return rf;
}

// Rows of `keys` (n device values) that the owner rule does not give to this rank
template <class Owner>
unsigned long long count_off_rank(b200vs_shard* sh, const long long* keys, int64_t n, Owner owner) {
  DevBuf<unsigned long long> bad;
  bad.reserve(1, 0, sh->ws);
  B200VS_CUDA(cudaMemsetAsync(bad.p, 0, 8, sh->ws));
  if (n) owner_check_kernel<<<(unsigned)cdiv(n, ROUTE_THREADS), ROUTE_THREADS, 0, sh->ws>>>(keys, n, sh->world, owner, sh->rank, bad.p);
  B200VS_CUDA(cudaGetLastError());
  unsigned long long h = 0;
  B200VS_CUDA(cudaMemcpyAsync(&h, bad.p, 8, cudaMemcpyDeviceToHost, sh->ws));
  B200VS_CUDA(cudaStreamSynchronize(sh->ws));
  return h;
}

// The list of every row [r0, r0 + n) of a rank file, on the device
void expand_lists(b200vs_shard* sh, const RankFile& rf, int64_t r0, int64_t n, DevBuf<long long>& d_off, long long* out) {
  d_off.reserve(rf.off.size(), 0, sh->ws);
  B200VS_CUDA(cudaMemcpyAsync(d_off.p, rf.off.data(), rf.off.size() * 8, cudaMemcpyHostToDevice, sh->ws));
  if (n) expand_lists_kernel<<<(unsigned)cdiv(n, 256), 256, 0, sh->ws>>>(d_off.p, rf.nlist(), r0, n, out);
  B200VS_CUDA(cudaGetLastError());
}

// Same world: every row of rank file rf must be owned by this rank (checked on the device).  graph_ids: HNSW, the labels of
// the saved graph.
void check_ownership(b200vs_shard* sh, const RankFile& rf, const std::vector<int64_t>& graph_ids) {
  const std::vector<int64_t>& ids = sh->ix->type == B200VS_HNSW ? graph_ids : rf.ids;
  const int64_t n = sh->rows ? (int64_t)ids.size() : rf.rows;
  DevBuf<long long> keys, d_off;
  keys.reserve((size_t)std::max<int64_t>(n, 1), 0, sh->ws);
  unsigned long long bad;
  if (sh->rows) {
    if (n) B200VS_CUDA(cudaMemcpyAsync(keys.p, ids.data(), (size_t)n * 8, cudaMemcpyHostToDevice, sh->ws));
    bad = count_off_rank(sh, keys.p, n, RowOwner{});
  } else {
    expand_lists(sh, rf, 0, n, d_off, keys.p);
    bad = count_off_rank(sh, keys.p, n, ListOwner{(rf.nlist() + sh->world - 1) / sh->world});
  }
  if (bad) fail(B200VS_EINTERNAL, rf.path + ": " + std::to_string(bad) + " rows belong to another rank (a rank file loaded on the wrong rank)");
}

struct PinnedBuf {
  unsigned char* p = nullptr;
  explicit PinnedBuf(size_t n) { B200VS_CUDA(cudaHostAlloc((void**)&p, std::max<size_t>(n, 1), cudaHostAllocDefault)); }
  ~PinnedBuf() { if (p) cudaFreeHost(p); }
};

void shard_load_locked(b200vs_shard* sh, const std::string& prefix) {
  IndexBase* ix = sh->ix;
  const int r = sh->rank, W2 = sh->world;
  cudaStream_t s = sh->ws;
  ix->set_device();
  check(agree(sh, attempt([&] {
    if (ix->count() + ix->deleted_count() > 0) fail(B200VS_EILLEGAL_PARAMETERS, "shard load needs an empty index on every rank");
  }), "shard load"));
  // 1) everything is checked before any index changes: the manifest against the index, every file this rank reads against
  //    the manifest, and (same world) the owner of every row
  ManifestHdr mh;
  std::vector<RankEntry> ents;
  std::vector<RankFile> files;
  std::vector<unsigned char> state;  // list-sharded: the snapshot's trained state; HNSW: the rank's graph
  check(agree(sh, attempt([&] {
    File f(prefix + ".manifest", "rb");
    f.read(&mh, sizeof(mh));
    if (memcmp(mh.magic, kManifestMagic, 8) != 0 || mh.version != kManifestVersion || mh.world < 1 || mh.world > ROUTE_MAX_WORLD)
      fail(B200VS_EINTERNAL, prefix + ".manifest: not a shard snapshot manifest");
    ents.resize((size_t)mh.world);
    f.read(ents.data(), ents.size() * sizeof(RankEntry));
    if (fgetc(f.f) != EOF) fail(B200VS_EINTERNAL, prefix + ".manifest: trailing bytes");
    ManifestHdr want = manifest_of(ix, mh.world);
    want.state_len = mh.state_len; want.state_digest = mh.state_digest;
    if (memcmp(&want, &mh, sizeof(mh)) != 0)
      fail(B200VS_EINTERNAL, "snapshot does not match this index (type / metric / dimension / creation parameters)");
    if (mh.world != W2 && ix->type == B200VS_HNSW)
      fail(B200VS_EVECTOR_NOT_SUPPORT, "an HNSW snapshot restores onto the same number of ranks only (a graph belongs to its rank)");
    if (!sh->rows && ix->is_trained()) {
      const std::vector<unsigned char> mine = state_of(ix);
      if ((int64_t)mine.size() != mh.state_len || digest_of(mine) != mh.state_digest)
        fail(B200VS_EINTERNAL, "the index's trained state differs from the snapshot's");
    }
    for (int fi = r; fi < mh.world; fi += W2) files.push_back(read_rank_file(ix, rank_path(prefix, fi, mh.world), ents[fi], mh, true));
    if (!sh->rows && mh.state_len > 0)
      state = files.empty() ? read_rank_file(ix, rank_path(prefix, 0, mh.world), ents[0], mh, false).state : files[0].state;
    std::vector<int64_t> graph_ids;
    if (ix->type == B200VS_HNSW) {
      state = files[0].state;
      if (!state.empty()) graph_ids = hnsw_state_labels(ix, state.data(), state.size());  // the labels of the saved graph
    }
    if (mh.world == W2) check_ownership(sh, files[0], graph_ids);
  }), "shard load"));
  // 2) the trained state: list-sharded, installed unless the index already holds it; HNSW, the graph
  check(agree(sh, attempt([&] {
    if (ix->type == B200VS_HNSW && !state.empty()) ix->set_state(state.data(), state.size());
    if (!sh->rows && !state.empty() && !ix->is_trained()) ix->set_state(state.data(), state.size());
  }), "shard load"));
  if (ix->type == B200VS_HNSW || (!sh->rows && mh.state_len == 0)) return;  // no rows to place
  // 3) list-sharded: every owned list pre-sized from the index-wide list lengths in one arena allocation (the binary lists
  //    grow as they are appended: a binary index has no list reservation)
  if (!sh->rows && !ix->binary()) {
    const int nlist = ix->nlist_now();
    std::vector<unsigned long long> mine((size_t)nlist, 0);
    for (const RankFile& rf : files)
      for (int l = 0; l < std::min(nlist, rf.nlist()); ++l) mine[l] += (unsigned long long)(rf.off[l + 1] - rf.off[l]);
    DevBuf<unsigned long long> d_cnt;
    d_cnt.reserve((size_t)nlist, 0, s);
    B200VS_CUDA(cudaMemcpyAsync(d_cnt.p, mine.data(), (size_t)nlist * 8, cudaMemcpyHostToDevice, s));
    std::vector<int64_t> cnt = sum_list_counts(sh, d_cnt.p, nlist);
    check(agree(sh, attempt([&] { reserve_owned_lists(sh, cnt); }), "shard load"));
  }
  // 4) rounds: each rank reads up to kRestoreChunkBytes of rows of its files into a pinned buffer and uploads them; the rows
  //    travel with their saved list (list-sharded) or by id (FLAT) through shard_add's routing, and the owner appends them
  //    exactly as stored: no coarse assignment, no normalisation, no encoding
  struct Chunk { size_t file; int64_t r0, n; };
  std::vector<Chunk> chunks;
  const int rb = restore_row_bytes(ix, mh);
  const int64_t per_chunk = std::max<int64_t>(1, (int64_t)kRestoreChunkBytes / rb);
  for (size_t fi = 0; fi < files.size(); ++fi)
    for (int64_t a = 0; a < files[fi].rows; a += per_chunk) chunks.push_back({fi, a, std::min(per_chunk, files[fi].rows - a)});
  const long long my_rounds = (long long)chunks.size();
  long long rounds = 0;
  for (const long long v : all_gather_host(sh, &my_rounds)) rounds = std::max(rounds, v);
  int64_t most = 0;
  for (const Chunk& c : chunks) most = std::max(most, c.n);
  PinnedBuf host((size_t)most * rb);
  DevBuf<unsigned char> d_rows;
  DevBuf<long long> d_ids, d_lists, d_off;
  for (long long k = 0; k < rounds; ++k) {
    Routed rv;
    int64_t n = 0;
    if (k < my_rounds) {
      const Chunk& c = chunks[(size_t)k];
      const RankFile& rf = files[c.file];
      n = c.n;
      File f(rf.path, "rb");
      if (fseeko(f.f, rf.rows_at + c.r0 * rb, SEEK_SET) != 0) fail(B200VS_EINTERNAL, "cannot seek in " + rf.path);
      f.read(host.p, (size_t)n * rb);
      d_rows.reserve((size_t)n * rb, 0, s); d_ids.reserve((size_t)n, 0, s); d_lists.reserve((size_t)n, 0, s);
      B200VS_CUDA(cudaMemcpyAsync(d_rows.p, host.p, (size_t)n * rb, cudaMemcpyHostToDevice, s));
      B200VS_CUDA(cudaMemcpyAsync(d_ids.p, rf.ids.data() + c.r0, (size_t)n * 8, cudaMemcpyHostToDevice, s));
      if (!sh->rows) expand_lists(sh, rf, c.r0, n, d_off, d_lists.p);
    }
    if (sh->rows) route_rows(sh, n, d_rows.p, rb, d_ids.p, nullptr, RowOwner{}, rv);
    else route_rows(sh, n, d_rows.p, rb, d_ids.p, d_lists.p, ListOwner{sh->lists_per_rank()}, rv);
    B200VS_CUDA(cudaStreamSynchronize(s));  // the pinned buffer and the sent rows are reused next round
    check(agree(sh, attempt([&] {
      if (rv.n) ix->add(AddReq::device(rv.n, rv.x.p, rv.ids.p, rv.lists.p, false, AddReq::ENCODED));
    }), "shard load"));
  }
}

// b200vs_shard_add[_device] (float rows) and b200vs_shard_add_binary[_device] (packed rows)
int shard_add(b200vs_shard* h, int64_t n, const void* x, const int64_t* ids, bool on_device, bool binary_call) {
  return guarded([&]() -> int {
    b200vs_shard* sh = get(h);
    check_row_type(sh, binary_call);
    if (n < 0 || (n > 0 && (!x || !ids))) fail(B200VS_EILLEGAL_PARAMETERS, "bad add arguments");
    std::lock_guard<Gate> g(sh->add_mu);
    if (on_device) {
      shard_add_impl(sh, n, x, (const long long*)ids, false, 0);
      return B200VS_OK;
    }
    sh->ix->set_device();
    DevBuf<unsigned char> dx;
    DevBuf<long long> di;
    upload_rows(sh, n, x, ids, dx, di);
    shard_add_impl(sh, n, dx.p, di.p, false, 0);
    return B200VS_OK;
  });
}

// ---------------------------------------------------------------------------------------------
// Rebuilds (b200vs_shard_need_rebuild / b200vs_shard_rebuild_from)
// ---------------------------------------------------------------------------------------------
// b200vs_need_rebuild's rule on the figures of the whole set: one all-gather of every rank's (live, tombstoned, trained);
// the caller holds add_mu.  IVF types: the set is trained when every rank is.
bool shard_need_rebuild_locked(b200vs_shard* sh) {
  IndexBase* ix = sh->ix;
  ix->set_device();
  long long mine[3];
  {
    std::shared_lock<std::shared_mutex> rl(ix->rw);
    mine[0] = (long long)ix->count(); mine[1] = (long long)ix->deleted_count(); mine[2] = ix->is_trained() ? 1 : 0;
  }
  const std::vector<long long> all = all_gather_host(sh, mine, 3);
  int64_t live = 0, dead = 0;
  bool trained = true;
  for (int w = 0; w < sh->world; ++w) {
    live += all[(size_t)w * 3]; dead += all[(size_t)w * 3 + 1]; trained = trained && all[(size_t)w * 3 + 2] != 0;
  }
  switch (ix->type) {
    case B200VS_IVF_FLAT:
    case B200VS_BINARY_IVF_FLAT: {  // shard_train refuses rather than degenerate nlist, so only nlist_org == 1 stays out
      const int64_t nlist_org = ix->params.nlist > 0 ? ix->params.nlist : 2048;
      return trained && nlist_org != 1 && live >= 256 * nlist_org && sh->train_rows_set <= live / 2;
    }
    case B200VS_IVF_PQ: return trained && live / 2 >= sh->train_rows_set;  // a set is in IVF-PQ mode (shard_create)
    case B200VS_HNSW: return dead > 0 && dead > (live + dead) / 2;       // nodes = live + tombstoned, halved on the sums
    default: return false;                                                // FLAT, BINARY_FLAT
  }
}

// The gates of a rebuild, taken in one order (by handle address) and released at scope exit: dst's exclusively, the source
// sets' shared.  Two rebuilds over overlapping sources (a split's child and parent, a merge beside a split of one of its
// sources) then never wait for each other on this rank; only the sources' writers wait for them.
struct RebuildGates {
  std::vector<std::pair<Gate*, bool>> held;  // (gate, exclusive), in the order taken
  RebuildGates(b200vs_shard* dst, const std::vector<b200vs_shard*>& srcs) {
    std::vector<b200vs_shard*> order(srcs);
    order.push_back(dst);
    std::sort(order.begin(), order.end(), std::less<b200vs_shard*>());
    for (b200vs_shard* sh : order) {
      const bool excl = sh == dst;
      if (excl) sh->add_mu.lock();
      else sh->add_mu.lock_shared();
      held.emplace_back(&sh->add_mu, excl);
    }
  }
  ~RebuildGates() {
    for (auto it = held.rbegin(); it != held.rend(); ++it) {
      if (it->second) it->first->unlock();
      else it->first->unlock_shared();
    }
  }
  RebuildGates(const RebuildGates&) = delete;
  RebuildGates& operator=(const RebuildGates&) = delete;
};

// The refusals of a set rebuild on this rank, decided before any index changes.  flat_ok: FLAT and BINARY_FLAT are served
// (b200vs_shard_rebuild_from_range).  Row-sharded sets: this rank's share of R is listed here, from the host bookkeeping,
// so that an HNSW dst too small for it and an id held by two sources are refused on every rank before any rank's dst changes
// (the per-rank rebuild that follows would find them only on the rank that holds them).
void check_shard_rebuild(b200vs_shard* dst, const std::vector<b200vs_shard*>& srcs, int64_t lo, int64_t hi, bool bad_range, bool flat_ok) {
  if (bad_range) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from_range: id_min > id_max");
  for (b200vs_shard* src : srcs)
    if (dst->world != src->world || dst->rank != src->rank) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from: dst and src differ in world or rank");
  IndexBase* d = dst->ix;
  {
    std::shared_lock<std::shared_mutex> rl(d->rw);
    for (b200vs_shard* src : srcs) check_rebuild_pair(*d, *src->ix);
  }
  if (!flat_ok && (d->type == B200VS_FLAT || d->type == B200VS_BINARY_FLAT)) fail(B200VS_EVECTOR_NOT_SUPPORT, "a Flat index never needs a rebuild");
  if (d->type == B200VS_IVF_PQ)
    fail(B200VS_EVECTOR_NOT_SUPPORT, "rebuild_from an IVF_PQ set: it stores only codes (rebuild it from host rows with shard_train + shard_add)");
  if (!dst->rows) return;
  std::vector<std::pair<int64_t, size_t>> r;  // (id, source) of this rank's share of R
  for (size_t k = 0; k < srcs.size(); ++k) {
    std::vector<int64_t> ids;
    {
      std::shared_lock<std::shared_mutex> rl(srcs[k]->ix->rw);
      srcs[k]->ix->live_ids(lo, hi, ids);
    }
    for (const int64_t id : ids) r.emplace_back(id, k);
  }
  if (d->type == B200VS_HNSW && d->params.max_elements > 0 && (int64_t)r.size() > d->params.max_elements)
    fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from: dst max_elements is below this rank's share of the rows");
  if (srcs.size() < 2) return;
  std::sort(r.begin(), r.end());
  for (size_t i = 1; i < r.size(); ++i)
    if (r[i].first == r[i - 1].first && r[i].second != r[i - 1].second)
      fail(B200VS_EVECTOR_ID_DUPLICATED, "rebuild_from_range: id " + std::to_string(r[i].first) + " is held by more than one source");
}

// List-sharded rebuild (IVF_FLAT, BINARY_IVF_FLAT), every step on dst's write stream and communicator.  Each source set in
// turn: its live rows with lo <= id <= hi in ascending id order (sorted_live_rows), routed to row_owner(id) (route_rows with
// RowOwner), so every row arrives in a block of its own source set.  Then one stable sort of what arrived, by id, over those
// blocks (a source set's block holds rank 0's rows first, each rank's in its own order, so ties keep (src rank, list-major
// position)); the sort's value carries the block, so an id that arrived from two source sets is refused there, after the
// routing has brought every copy of it to one rank.  Then shard_train's flow and shard_add's flow on those device rows.
// Every local step before a collective (the sorts, the routing's and the add's copies, the k-means, the state install, the
// add) is agreed, so a device failure on one rank, an allocation that does not fit included, is returned by every rank.
// Returns the live rows this rank's dst holds.
int64_t shard_rebuild_lists(b200vs_shard* dst, const std::vector<b200vs_shard*>& srcs, int64_t lo, int64_t hi, const char* what) {
  IndexBase* d = dst->ix;
  const int words = d->binary() ? (d->dim / 8 + 3) / 4 : d->dim;
  const cudaStream_t ws = dst->ws;
  d->set_device();
  // 1, 2) each source set's rows in the range sorted by id, behind every write its own stream holds, then to the training
  // owner (the routing's send and receive copies are reserved in agreed steps); the sorted copy dies once routed
  std::vector<Routed> rv(srcs.size());
  for (size_t k = 0; k < srcs.size(); ++k) {
    IndexBase* s = srcs[k]->ix;
    DevBuf<uint32_t> rows;
    DevBuf<long long> ids;
    int64_t n = 0;
    check(agree(dst, attempt([&] {
      std::shared_lock<std::shared_mutex> rl(s->rw);
      B200VS_CUDA(cudaStreamSynchronize(s->stream));
      n = sorted_live_rows(d, {s}, lo, hi, words, rows, ids, ws);
    }), what));
    route_rows(dst, n, rows.p, words * 4, ids.p, nullptr, RowOwner{}, rv[k], true);
    local_step(dst, true, what, [&] { B200VS_CUDA(cudaStreamSynchronize(ws)); });  // the sent copy is read before rows die
  }
  // 3) stable sort of what arrived by id over the source blocks: rows_r; an id from two source sets is refused
  DevBuf<uint32_t> tx;
  DevBuf<long long> tids;
  int64_t m = 0;
  std::vector<DeviceRows> blocks;
  for (const Routed& b : rv) {
    blocks.push_back({b.n, b.ids.p, reinterpret_cast<const uint32_t*>(b.x.p)});
    m += b.n;
  }
  check(agree(dst, attempt([&] { sorted_live_rows(d, blocks, words, tx, tids, ws); }), what));
  rv.clear();
  int64_t total = 0;
  for (const long long c : all_gather_host(dst, &m)) total += c;
  if (total == 0) return 0;  // nothing live anywhere: dst stays untrained
  // 4, 5) the rank-local coarse k-means, the centroid all-gather, the state install (refuses a rank below nlist / world rows)
  shard_train_locked(dst, m, m ? tx.p : nullptr, true);
  // 6) the collective add of rows_r: binary rows go back to their packed dim / 8 bytes
  const void* xa = tx.p;
  DevBuf<unsigned char> packed;
  const size_t nb = d->query_row_bytes();
  local_step(dst, true, what, [&] {
    if (!d->binary() || nb == (size_t)words * 4 || !m) return;
    packed.reserve((size_t)m * nb, 0, ws);
    B200VS_CUDA(cudaMemcpy2DAsync(packed.p, nb, tx.p, (size_t)words * 4, nb, (size_t)m, cudaMemcpyDeviceToDevice, ws));
    B200VS_CUDA(cudaStreamSynchronize(ws));
    tx.free();
    xa = packed.p;
  });
  shard_add_impl(dst, m, xa, tids.p, false, 0, true);
  std::shared_lock<std::shared_mutex> rl(d->rw);
  return d->count();
}

// The body of b200vs_shard_rebuild_from[_range] once the arguments are checked: fill dst from the live rows with
// lo <= id <= hi of the source sets srcs.  The gates come first, then the agreed refusals; row-sharded sets run the
// single-index rebuild of each rank's sources into its dst index, then one more agreement.  Returns the live rows this
// rank's dst holds.
int64_t shard_rebuild(b200vs_shard* dst, const std::vector<b200vs_shard*>& srcs, int64_t lo, int64_t hi, bool bad_range, bool flat_ok,
                      const char* what) {
  RebuildGates gates(dst, srcs);
  dst->ix->set_device();
  check(agree(dst, attempt([&] { check_shard_rebuild(dst, srcs, lo, hi, bad_range, flat_ok); }), what));
  if (!dst->rows) return shard_rebuild_lists(dst, srcs, lo, hi, what);
  std::vector<IndexBase*> ixs;
  for (b200vs_shard* src : srcs) ixs.push_back(src->ix);
  int64_t n = 0;
  check(agree(dst, attempt([&] { n = rebuild_range(dst->ix, ixs, lo, hi, true); }), what));
  return n;
}

}  // namespace

extern "C" {

// Collective: every rank passes the rows IT holds (any rows; n may differ per rank, 0 allowed); each row is assigned to its
// nearest centroid and travels to the rank that owns that list (grouped ncclSend / ncclRecv over NVLink).
int b200vs_shard_add_device(b200vs_shard* h, int64_t n, const float* x_dev, const int64_t* ids_dev) {
  return shard_add(h, n, x_dev, ids_dev, true, false);
}
int b200vs_shard_add_binary_device(b200vs_shard* h, int64_t n, const uint8_t* x_dev, const int64_t* ids_dev) {
  return shard_add(h, n, x_dev, ids_dev, true, true);
}
int b200vs_shard_add(b200vs_shard* h, int64_t n, const float* x, const int64_t* ids) { return shard_add(h, n, x, ids, false, false); }
int b200vs_shard_add_binary(b200vs_shard* h, int64_t n, const uint8_t* x, const int64_t* ids) { return shard_add(h, n, x, ids, false, true); }

// Collective batched HNSW build of a row-sharded HNSW index: shard_add's routing, then b200vs_hnsw_add_batched with `batch`
// on the rows each rank received, in arrival order.
int b200vs_shard_hnsw_add_batched(b200vs_shard* h, int64_t n, const float* x, const int64_t* ids, int32_t batch) {
  return guarded([&]() -> int {
    b200vs_shard* sh = get(h);
    if (sh->ix->type != B200VS_HNSW) fail(B200VS_EILLEGAL_PARAMETERS, "batched HNSW construction needs an HNSW index");
    if (n < 0 || (n > 0 && (!x || !ids))) fail(B200VS_EILLEGAL_PARAMETERS, "bad add arguments");
    std::lock_guard<Gate> g(sh->add_mu);
    sh->ix->set_device();
    DevBuf<unsigned char> dx;
    DevBuf<long long> di;
    upload_rows(sh, n, x, ids, dx, di);
    shard_add_impl(sh, n, dx.p, di.p, true, batch);
    return B200VS_OK;
  });
}

// Collective snapshot of the sharded index under `prefix` (every rank passes the same prefix, a path every rank can reach).
int b200vs_shard_save(b200vs_shard* h, const char* prefix) {
  return guarded([&]() -> int {
    b200vs_shard* sh = get(h);
    if (!prefix || !*prefix) fail(B200VS_EILLEGAL_PARAMETERS, "null snapshot prefix");
    std::lock_guard<Gate> g(sh->add_mu);
    shard_save_locked(sh, prefix);
    return B200VS_OK;
  });
}

// Collective restore of a snapshot into the empty indexes of this shard, onto the same or (not HNSW) another world size.
int b200vs_shard_load(b200vs_shard* h, const char* prefix) {
  return guarded([&]() -> int {
    b200vs_shard* sh = get(h);
    if (!prefix || !*prefix) fail(B200VS_EILLEGAL_PARAMETERS, "null snapshot prefix");
    std::lock_guard<Gate> g(sh->add_mu);
    shard_load_locked(sh, prefix);
    if (!sh->rows) sh->train_rows_set = live_rows_set(sh);
    return B200VS_OK;
  });
}

// Collective NeedToRebuild of the whole set: 1, 0, or a status negated; the same answer on every rank.
int b200vs_shard_need_rebuild(b200vs_shard* h) {
  int r = 0;
  const int rc = guarded([&]() -> int {
    b200vs_shard* sh = get(h);
    std::lock_guard<Gate> g(sh->add_mu);
    r = shard_need_rebuild_locked(sh) ? 1 : 0;
    return B200VS_OK;
  });
  return rc == B200VS_OK ? r : -rc;
}

// Collective rebuild of the fresh set dst from the set src (every rank passes its own dst and src): the one-source,
// every-id case of b200vs_shard_rebuild_from_range, with FLAT and BINARY_FLAT refused.
int b200vs_shard_rebuild_from(b200vs_shard* dst_h, b200vs_shard* src_h, int64_t* n_rows) {
  return guarded([&]() -> int {
    if (n_rows) *n_rows = 0;
    b200vs_shard* dst = get(dst_h);
    b200vs_shard* src = get(src_h);
    if (dst == src) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from: dst and src are the same shard");
    const int64_t n = shard_rebuild(dst, {src}, 0, INT64_MAX, false, false, "shard rebuild_from");
    if (n_rows) *n_rows = n;
    return B200VS_OK;
  });
}

// Collective split / merge rebuild of the fresh set dst from the live rows with id_min <= id < id_max of the source sets
// srcs[0 .. n_src) (every rank passes its own dst and its own rank's source shards).  The argument errors are refused here,
// on the rank that meets them, before any collective.
int b200vs_shard_rebuild_from_range(b200vs_shard* dst_h, int32_t n_src, b200vs_shard* const* srcs_h, int64_t id_min, int64_t id_max,
                                    int64_t* n_rows) {
  return guarded([&]() -> int {
    if (n_rows) *n_rows = 0;
    if (n_src < 1 || n_src > kRebuildMaxSources || !srcs_h)
      fail(B200VS_EILLEGAL_PARAMETERS, "shard rebuild_from_range: 1 to 16 sources, in a non-null list");
    b200vs_shard* dst = get(dst_h);
    std::vector<b200vs_shard*> srcs;
    for (int32_t i = 0; i < n_src; ++i) {
      b200vs_shard* src = get(srcs_h[i]);
      if (src == dst) fail(B200VS_EILLEGAL_PARAMETERS, "shard rebuild_from_range: dst is among the sources");
      if (std::find(srcs.begin(), srcs.end(), src) != srcs.end()) fail(B200VS_EILLEGAL_PARAMETERS, "shard rebuild_from_range: a source is listed twice");
      srcs.push_back(src);
    }
    // [id_min, id_max) as inclusive bounds; id_max - 1 cannot overflow once the range holds an id
    const bool none = id_min >= id_max;
    const int64_t n = shard_rebuild(dst, srcs, none ? 1 : id_min, none ? 0 : id_max - 1, id_min > id_max, true, "shard rebuild_from_range");
    if (n_rows) *n_rows = n;
    return B200VS_OK;
  });
}

// Owner of every id of a row-sharded index (pure host function): callers place rows where they belong so they travel nowhere.
int b200vs_row_owner(int32_t world, int64_t n, const int64_t* ids, int32_t* out_rank) {
  return guarded([&]() -> int {
    if (world < 1 || world > ROUTE_MAX_WORLD || n < 0 || (n > 0 && (!ids || !out_rank)))
      fail(B200VS_EILLEGAL_PARAMETERS, "bad row_owner arguments (world must be in [1, 1024])");
    for (int64_t i = 0; i < n; ++i) out_rank[i] = row_owner_of((long long)ids[i], world);
    return B200VS_OK;
  });
}

// Collective delete (VectorIndexIvfFlat::Delete, vector_index_ivf_flat.cc:162-189, over all shards): every rank passes the same
// id list and drops the rows it holds; the removed counts are summed over the ranks.  "remove not found vector id" ->
// EVECTOR_INVALID only when NO rank held any of the ids (:180-184).  Upsert of a sharded index = this call (a not-found
// status ignored), then b200vs_shard_add*: the new row may live on another rank than the old one.  Row-sharded FLAT and
// HNSW follow their single-index rule instead: unknown ids are ignored and the status is OK.
int b200vs_shard_remove_ids(b200vs_shard* h, int64_t n, const int64_t* ids, int64_t* n_removed) {
  return guarded([&]() -> int {
    b200vs_shard* sh = get(h);
    if (n_removed) *n_removed = 0;
    if (n <= 0) return B200VS_OK;  // "delete_ids.empty() -> OK"
    if (!ids) fail(B200VS_EILLEGAL_PARAMETERS, "null ids");
    std::lock_guard<Gate> g(sh->add_mu);
    IndexBase* ix = sh->ix;
    const int64_t local = ix->remove(n, ids);  // -1: untrained (OK, nothing to do)
    ix->set_device();
    long long removed = 0;
    bool untrained = false;
    for (const int64_t v : all_gather_host(sh, &local)) {
      if (v > 0) removed += v;
      untrained |= v < 0;
    }
    if (n_removed) *n_removed = removed;
    if (!sh->rows && removed == 0 && !untrained) fail(B200VS_EVECTOR_INVALID, "remove not found vector id");
    return B200VS_OK;
  });
}

// Bulk builds of large shards: first pass every chunk through plan_add (assignment only, rows are NOT stored), then
// plan_commit all-reduces the per-list counts and pre-sizes the owned lists in one arena allocation; the second pass
// (b200vs_shard_add*) then never relocates a list or re-allocates the arena.
int b200vs_shard_plan_add_device(b200vs_shard* h, int64_t n, const float* x_dev) {
  return guarded([&]() -> int {
    b200vs_shard* sh = get(h);
    if (sh->ix->binary()) fail(B200VS_EVECTOR_NOT_SUPPORT, "a binary index has no list pre-sizing");
    if (sh->rows) fail(B200VS_EVECTOR_NOT_SUPPORT, "a row-sharded index has no inverted lists to pre-size");
    if (n <= 0 || !x_dev) fail(B200VS_EILLEGAL_PARAMETERS, "bad plan arguments");
    std::lock_guard<Gate> g(sh->add_mu);
    IndexBase* ix = sh->ix;
    ix->set_device();
    const int nlist = ix->nlist_now();
    if (!sh->planning) {
      sh->plan_counts.reserve((size_t)nlist, 0, sh->ws);
      B200VS_CUDA(cudaMemsetAsync(sh->plan_counts.p, 0, (size_t)nlist * 8, sh->ws));
      sh->planning = true;
    }
    DevBuf<float> prep;
    DevBuf<long long> lists;
    assign_rows(sh, n, x_dev, prep, lists);
    count_lists_kernel<<<(unsigned)cdiv(n, 256), 256, 0, sh->ws>>>(lists.p, n, nlist, sh->plan_counts.p);
    B200VS_CUDA(cudaGetLastError());
    B200VS_CUDA(cudaStreamSynchronize(sh->ws));
    return B200VS_OK;
  });
}

int b200vs_shard_plan_commit(b200vs_shard* h) {
  return guarded([&]() -> int {
    b200vs_shard* sh = get(h);
    if (sh->ix->binary()) fail(B200VS_EVECTOR_NOT_SUPPORT, "a binary index has no list pre-sizing");
    if (sh->rows) fail(B200VS_EVECTOR_NOT_SUPPORT, "a row-sharded index has no inverted lists to pre-size");
    std::lock_guard<Gate> g(sh->add_mu);
    IndexBase* ix = sh->ix;
    ix->set_device();
    const int nlist = ix->nlist_now();
    if (!sh->planning) {
      sh->plan_counts.reserve((size_t)nlist, 0, sh->ws);
      B200VS_CUDA(cudaMemsetAsync(sh->plan_counts.p, 0, (size_t)nlist * 8, sh->ws));
    }
    std::vector<int64_t> cnt = sum_list_counts(sh, sh->plan_counts.p, nlist);
    sh->planning = false;
    reserve_owned_lists(sh, cnt);
    return B200VS_OK;
  });
}

int b200vs_shard_search_device(b200vs_shard* h, int64_t seq, int64_t nq, const float* xq_dev, int32_t k, const b200vs_search_params* sp,
                               float* out_dist_dev, int64_t* out_ids_dev, void* stream) {
  return shard_read(h, {READ_TOPK, false, true, stream, seq, nq, xq_dev, 0.f, k, sp, out_dist_dev, out_ids_dev, nullptr});
}
int b200vs_shard_search_binary_device(b200vs_shard* h, int64_t seq, int64_t nq, const uint8_t* xq_dev, int32_t k,
                                      const b200vs_search_params* sp, float* out_dist_dev, int64_t* out_ids_dev, void* stream) {
  return shard_read(h, {READ_TOPK, true, true, stream, seq, nq, xq_dev, 0.f, k, sp, out_dist_dev, out_ids_dev, nullptr});
}

int b200vs_shard_search(b200vs_shard* h, int64_t seq, int64_t nq, const float* xq, int32_t k, const b200vs_search_params* sp, float* out_dist,
                        int64_t* out_ids) {
  return shard_read(h, {READ_TOPK, false, false, nullptr, seq, nq, xq, 0.f, k, sp, out_dist, out_ids, nullptr});
}
int b200vs_shard_search_binary(b200vs_shard* h, int64_t seq, int64_t nq, const uint8_t* xq, int32_t k, const b200vs_search_params* sp,
                               float* out_dist, int64_t* out_ids) {
  return shard_read(h, {READ_TOPK, true, false, nullptr, seq, nq, xq, 0.f, k, sp, out_dist, out_ids, nullptr});
}

int b200vs_shard_search_deep(b200vs_shard* h, int64_t seq, int64_t nq, const float* xq, int32_t k, const b200vs_search_params* sp,
                             float* out_dist, int64_t* out_ids) {
  return shard_read(h, {READ_DEEP, false, false, nullptr, seq, nq, xq, 0.f, k, sp, out_dist, out_ids, nullptr});
}
int b200vs_shard_search_binary_deep(b200vs_shard* h, int64_t seq, int64_t nq, const uint8_t* xq, int32_t k, const b200vs_search_params* sp,
                                    float* out_dist, int64_t* out_ids) {
  return shard_read(h, {READ_DEEP, true, false, nullptr, seq, nq, xq, 0.f, k, sp, out_dist, out_ids, nullptr});
}

int b200vs_shard_range_search_device(b200vs_shard* h, int64_t seq, int64_t nq, const float* xq_dev, float radius, int32_t max_results,
                                     const b200vs_search_params* sp, float* out_dist_dev, int64_t* out_ids_dev, int32_t* out_counts_dev,
                                     void* stream) {
  return shard_read(h, {READ_RANGE, false, true, stream, seq, nq, xq_dev, radius, max_results, sp, out_dist_dev, out_ids_dev, out_counts_dev});
}
int b200vs_shard_range_search_binary_device(b200vs_shard* h, int64_t seq, int64_t nq, const uint8_t* xq_dev, float radius,
                                            int32_t max_results, const b200vs_search_params* sp, float* out_dist_dev, int64_t* out_ids_dev,
                                            int32_t* out_counts_dev, void* stream) {
  return shard_read(h, {READ_RANGE, true, true, stream, seq, nq, xq_dev, radius, max_results, sp, out_dist_dev, out_ids_dev, out_counts_dev});
}

int b200vs_shard_range_search(b200vs_shard* h, int64_t seq, int64_t nq, const float* xq, float radius, int32_t max_results,
                              const b200vs_search_params* sp, float* out_dist, int64_t* out_ids, int32_t* out_counts) {
  return shard_read(h, {READ_RANGE, false, false, nullptr, seq, nq, xq, radius, max_results, sp, out_dist, out_ids, out_counts});
}
int b200vs_shard_range_search_binary(b200vs_shard* h, int64_t seq, int64_t nq, const uint8_t* xq, float radius, int32_t max_results,
                                     const b200vs_search_params* sp, float* out_dist, int64_t* out_ids, int32_t* out_counts) {
  return shard_read(h, {READ_RANGE, true, false, nullptr, seq, nq, xq, radius, max_results, sp, out_dist, out_ids, out_counts});
}

}  // extern "C"
