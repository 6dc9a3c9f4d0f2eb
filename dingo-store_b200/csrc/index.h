// index.h — host-side index objects of libb200vs (device memory owners + search orchestration).
//
// One object per dingo-store vector index (= per Raft region, src/vector/vector_index.h:54-55).  These are
// the GPU replacements of the faiss / hnswlib objects the reference plugins own
// (index_id_map2_ flat.cc:98, index_ ivf_flat.cc:809-816, raw_ivf_pq.cc:554-564, hnsw_index_ hnsw.cc:181).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <cstring>
#include <functional>
#include <mutex>
#include <new>
#include <shared_mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/b200vs.h"
#include "common.cuh"
#include "deep_select.cuh"
#include "snapshot.h"

namespace b200vs {

struct StatusError {
  int code;
  std::string msg;
};
[[noreturn]] inline void fail(int code, const std::string& m) { throw StatusError{code, m}; }

// Vector ids are non-negative: every scan, the oracle and the shard merge read a negative id as a tombstone or an empty
// result slot.  Every add refuses a batch holding one before it changes anything.
inline void check_ids_nonnegative(int64_t n, const int64_t* ids) {
  for (int64_t i = 0; i < n; ++i)
    if (ids[i] < 0) fail(B200VS_EILLEGAL_PARAMETERS, "vector id is negative: " + std::to_string(ids[i]));
}

// The body of every extern "C" entry point: no exception leaves the library, each failure becomes a b200vs_status and
// b200vs_last_error's text.
template <class F>
int guarded(F&& f) {
  try {
    return f();
  } catch (const StatusError& e) {
    g_last_error = e.msg;
    return e.code;
  } catch (const CudaError& e) {
    g_last_error = e.what();
    return B200VS_EINTERNAL;
  } catch (const std::bad_alloc&) {
    g_last_error = "out of host memory";
    return B200VS_EINTERNAL;
  } catch (const std::exception& e) {
    g_last_error = e.what();
    return B200VS_EINTERNAL;
  } catch (...) {
    g_last_error = "unknown error";
    return B200VS_EINTERNAL;
  }
}

template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;  // elements
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
  void free() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  void swap(DevBuf& o) { std::swap(p, o.p); std::swap(cap, o.cap); }
  // grow to >= n elements; keeps the first `keep` elements (copied on `s`)
  void reserve(size_t n, size_t keep, cudaStream_t s) {
    if (!try_reserve(n, keep, s)) throw CudaError("cudaMalloc of " + std::to_string(n * sizeof(T)) + " B failed: out of memory");
  }
  // reserve() that returns false, changing nothing, when the device is out of memory.  The failed allocation is cleared
  // from the runtime's last error, so a later cudaGetLastError() check does not report it again.
  bool try_reserve(size_t n, size_t keep, cudaStream_t s) {
    if (n <= cap) return true;
    T* np = nullptr;
    const cudaError_t e = cudaMalloc(&np, n * sizeof(T));
    if (e == cudaErrorMemoryAllocation) { cudaGetLastError(); return false; }
    B200VS_CUDA(e);
    if (keep && p) B200VS_CUDA(cudaMemcpyAsync(np, p, keep * sizeof(T), cudaMemcpyDeviceToDevice, s));
    if (p) { B200VS_CUDA(cudaStreamSynchronize(s)); cudaFree(p); }
    p = np; cap = n;
    return true;
  }
};

// bump allocator for per-search scratch; reset at the start of every search (searches on one index are
// serialised by gpu_mu and stream-ordered, so reuse is safe)
struct Scratch {
  DevBuf<unsigned char> buf;
  size_t used = 0;
  std::vector<std::pair<void*, size_t>> overflow;  // extra cudaMalloc blocks when buf is too small
  size_t peak_overflow = 0;                        // most overflow bytes alive at once since the last reset
  ~Scratch() { release_overflow(); }
  void release_overflow() { for (auto& o : overflow) cudaFree(o.first); overflow.clear(); }
  size_t overflow_bytes() const { size_t b = 0; for (auto& o : overflow) b += o.second + 256; return b; }
  void reset(cudaStream_t s) {
    peak_overflow = std::max(peak_overflow, overflow_bytes());
    if (peak_overflow) {  // grow the main buffer so the next search fits without overflow blocks
      B200VS_CUDA(cudaStreamSynchronize(s));
      release_overflow();
      size_t want = (buf.cap + peak_overflow) * 3 / 2;
      peak_overflow = 0;
      buf.free();
      buf.reserve(want, 0, s);
    }
    used = 0;
  }
  template <class T>
  T* alloc(size_t n) {
    size_t bytes = (n * sizeof(T) + 255) / 256 * 256;
    if (used + bytes <= buf.cap) { T* r = reinterpret_cast<T*>(buf.p + used); used += bytes; return r; }
    void* p = nullptr;
    B200VS_CUDA(cudaMalloc(&p, bytes));
    overflow.emplace_back(p, bytes);
    return reinterpret_cast<T*>(p);
  }
  // scoped reuse inside one operation (chunk loops): everything allocated after mark() is handed back by release().
  // Overflow blocks taken in between are freed (cudaFree waits for the device), so a loop over many chunks holds one
  // chunk's worth of memory, not the sum.
  struct Mark { size_t used, nover; };
  Mark mark() const { return Mark{used, overflow.size()}; }
  void release(const Mark& m) {
    peak_overflow = std::max(peak_overflow, overflow_bytes());
    while (overflow.size() > m.nover) { cudaFree(overflow.back().first); overflow.pop_back(); }
    used = m.used;
  }
};

// A lane = one in-flight search: its own scratch arena, serialised by its own mutex, stream-ordered.  Several lanes let
// concurrent callers (the reference issues searches from a 16-thread pool, src/server/server.cc:868-873) overlap on the
// GPU: the small kernels of one batch run under the HBM-bound list scan of another.  A lane that moves to another
// stream is ordered behind its previous search with an event (device-side wait, the host never blocks).
struct Lane {
  Scratch s;
  std::mutex mu;
  std::atomic<cudaStream_t> last{nullptr};  // stream of the lane's previous search
  cudaStream_t own = nullptr;               // lane-owned stream for host-pointer / NULL-stream calls
  cudaEvent_t done = nullptr;               // recorded behind the lane's latest search
  std::atomic<bool> done_valid{false};
  unsigned long long tick = 0;              // last use (lane_pick_mu), for least-recently-used hand-out
};
constexpr int kLanes = 8;

// Request coalescing for host-pointer searches (SURVEY 8b: "b200vs_search internally coalesces concurrent callers").  The
// unchanged reference caller slices every batch into single-query tasks on a 16-thread pool (src/vector/vector_index.cc:54,
// :244-271), so the plugin sees many concurrent nq = 1 calls.  Callers queue here; the one that finds no leader active
// becomes the leader, takes every compatible pending request (same k / nprobe / efsearch / exact_only, no id filters) and
// runs them as ONE batch — large enough batches reach the tensor-core tile path — then hands the results back.  Float
// and binary indexes share it: a request's queries are nq rows of the index's query_row_bytes().
struct CoalesceReq {
  int64_t nq = 0;
  const void* xq = nullptr;
  int k = 0;
  b200vs_search_params sp{};
  float* out_dist = nullptr;
  int64_t* out_ids = nullptr;
  int rc = 0;
  std::string err;
  bool done = false;
};
struct Coalescer {
  std::mutex mu;
  std::condition_variable cv;
  std::vector<CoalesceReq*> pending;
  bool busy = false;
  std::atomic<int> enabled{1};
  std::atomic<int64_t> batches{0}, requests{0};  // statistics: leader batches run / requests served through them
};

struct SearchCtx {  // resolved per-search parameters, device filter included
  int nprobe = 0;
  int efsearch = 0;
  int exact_only = 0;
  int has_range = 0, negate = 0;
  long long rmin = 0, rmax = 0;
  const long long* sorted_ids_dev = nullptr;
  long long n_ids = 0;
  bool has_filter() const { return has_range || sorted_ids_dev; }
};
struct IndexBase;
struct TcView;
// resolve search params; uploads the sorted id list into the calling lane's scratch (stream-ordered on s)
SearchCtx make_ctx(IndexBase* ix, const b200vs_search_params* sp, cudaStream_t s);

// One read of an index (IndexBase::search).  Every pointer is on the index's device.
struct SearchReq {
  int64_t nq = 0;
  const void* xq = nullptr;           // query rows: FP32, or packed bits (dim / 8 bytes) on a binary index
  bool prepared = false;              // FP32 rows already normalised for cosine
  const long long* probes = nullptr;  // the caller's probe table [nq, nprobe] (IVF types); null = the index's own coarse pass
  int nprobe = 0;
  int k = 0;                          // top-k, or max_results when range
  bool range = false;                 // range search: the hits inside radius, closest first, at most k of them
  float radius = 0.f;
  bool deep = false;                  // top-k through the deep path (run_deep): any k up to kDeepMaxK, always exact
  bool raw = false;                   // od = the raw metric value (L2 distance | ip), the key the single-index select ranks
                                      // by and a merge of several indexes' results has to order by, instead of the API distance
  const SearchCtx* sc = nullptr;
  float* od = nullptr;                // [nq, k]
  long long* oi = nullptr;            // [nq, k], -1 past the last result
  int* oc = nullptr;                  // [nq] hits per query (range)
  const float* fq() const { return static_cast<const float*>(xq); }
};
// the results of a search that finds nothing (an untrained or empty index): ids -1, distances 0, range counts 0
void fill_empty(const SearchReq& r, cudaStream_t s);
// The search of one Flat view (tc_scan.cuh): a Flat index's rows, or every row slot of another index for a brute-force scan.
// Top-k through the tile scan, the one-query kernel or the exact scan, deep top-k through the deep path, range through the
// tile scan or the exact scan; every path selects the same rows (index.cu).
void flat_view_search(IndexBase* ix, const TcView& v, const SearchReq& r, cudaStream_t s);
// b200vs_brute_force_search / b200vs_brute_force_range_search (brute_force.cu): r over every row ix->brute_force_rows gives,
// with the results b200vs_scan_* / b200vs_scan_range_* return for those rows fed in ascending id order.
void brute_force(IndexBase* ix, const SearchReq& r, cudaStream_t s);

// One write of rows into an index (IndexBase::add).  Host rows come with host ids; device rows (on the index's device) come
// with device ids, and with the same ids on the host when the caller already holds them.
struct AddReq {
  enum Form {
    RAW,       // the caller's rows: the index applies its own cosine rule
    PREPARED,  // stored exactly as given (already normalised for cosine): a snapshot restore, a routed shard row, a rebuild
    ENCODED,   // the rows as export_lists writes them: IVF-PQ code rows (code_size bytes each); PREPARED on every other type
  };
  int64_t n = 0;
  const void* x = nullptr;              // rows in the index's row format: FP32, packed bits (dim / 8 bytes), or code rows
  bool on_device = false;               // x, ids_dev and lists are on the index's device
  const int64_t* ids = nullptr;         // host ids: always for host rows; optional beside device rows
  const long long* ids_dev = nullptr;   // device ids of device rows
  const long long* lists = nullptr;     // device rows: the caller's inverted list of every row (IVF types); null = the nearest
  bool upsert = false;
  Form form = RAW;
  bool batched = false;                 // HNSW: the batched GPU build (b200vs_hnsw_add_batched) with `batch` rows per batch
  int batch = 0;                        // 0 = the library default
  static AddReq host(int64_t n, const void* x, const int64_t* ids, bool upsert = false, Form form = RAW) {
    AddReq r;
    r.n = n; r.x = x; r.ids = ids; r.upsert = upsert; r.form = form;
    return r;
  }
  static AddReq device(int64_t n, const void* x, const long long* ids_dev, const long long* lists = nullptr, bool upsert = false,
                       Form form = RAW) {
    AddReq r;
    r.n = n; r.x = x; r.on_device = true; r.ids_dev = ids_dev; r.lists = lists; r.upsert = upsert; r.form = form;
    return r;
  }
};

// One source of a rebuild (b200vs_rebuild_from[_range], IndexBase::live_rows): the live rows of an index inside an id range,
// as their ids and row slots in the index's storage order from its host bookkeeping, and the device row store they index.
constexpr int kRebuildMaxSources = 16;
struct RebuildSource {
  std::vector<int64_t> ids;
  std::vector<long long> slots;
  const uint32_t* rows = nullptr;            // the row store: the same number of 32-bit words per row in every source
  cudaStream_t stream = nullptr;             // the stream the store's writes run on
  std::shared_lock<std::shared_mutex> hold;  // the reader lock of an inner index whose writers do not take the outer one
};

// The header of IndexBase::save's container ("B2VSIDX1" / "B2VSBIN1"), followed by the trained-state blob (state_len
// bytes), the list offsets (nlist + 1 int64), the ids (count int64) and the rows (count rows, list-major).
struct IndexFileHdr { char magic[8]; int32_t type, metric, dim, nlist; int64_t state_len, count; };

struct IndexBase {
  b200vs_type type;
  b200vs_metric metric;
  int dim;
  int device;
  b200vs_params params;
  cudaStream_t stream = nullptr;
  cudaStream_t last_stream = nullptr;
  std::shared_mutex rw;  // readers = searches, writers = add/remove/train (reference RWLock)
  std::mutex gpu_mu;     // writers / maintenance (they also hold rw exclusively)
  Lane lanes[kLanes];
  Coalescer coalescer;
  std::atomic<unsigned> lane_rr{0};
  std::mutex lane_pick_mu;
  unsigned long long lane_tick = 0;
  static thread_local Lane* tl_lane;       // the calling thread's active lane (set by LaneGuard)
  static thread_local IndexBase* tl_owner;
  Lane& cur() { return (tl_owner == this && tl_lane) ? *tl_lane : lanes[0]; }
  // wait for the asynchronous work of every earlier search (device-pointer searches return before the GPU is done);
  // writers call it before touching index memory or the lane-0 scratch
  void quiesce() { for (auto& l : lanes) if (l.done_valid.load()) cudaEventSynchronize(l.done); }
  struct ScratchProxy {  // `ix->scratch.alloc<T>(n)` resolves to the calling thread's lane
    IndexBase* ix;
    template <class T> T* alloc(size_t n) { return ix->cur().s.alloc<T>(n); }
    void reset(cudaStream_t st) { ix->cur().s.reset(st); }
    Scratch::Mark mark() { return ix->cur().s.mark(); }
    void release(const Scratch::Mark& m) { ix->cur().s.release(m); }
  } scratch{this};
  // counters of the LAST search; several lanes may search at once, so they are relaxed atomics (the values of two
  // overlapping searches interleave — they are diagnostics — but there is no data race)
  std::atomic<int64_t> stats[8] = {};
  // profiling only (one caller at a time): CUDA-event marks between the phases of a search, b200vs_last_phase_times
  enum Phase { PH_COARSE_PREP = 0, PH_COARSE_SCAN, PH_COARSE_FINAL, PH_PLAN, PH_SAMPLE, PH_TAU, PH_CAPTURE, PH_FINAL, PH_FALLBACK, PH_OTHER, PH_COMM, PH_MERGE,
               PH_BUILD_SEARCH, PH_BUILD_SELECT, PH_BUILD_LINK,  // b200vs_hnsw_add_batched: construction search / forward links / reverse links
               PH_COUNT };
  float phase_ms[PH_COUNT] = {0};
  std::vector<std::pair<int, cudaEvent_t>> phase_marks;
  void phase(int id, cudaStream_t s) {  // "phase id starts here"
    if (!profiling) return;
    cudaEvent_t e = nullptr;
    if (cudaEventCreate(&e) != cudaSuccess) return;
    cudaEventRecord(e, s);
    phase_marks.emplace_back(id, e);
  }
  void phases_finish(cudaStream_t s) {
    if (phase_marks.empty()) return;
    phase(-1, s);
    cudaEventSynchronize(phase_marks.back().second);
    for (size_t i = 0; i + 1 < phase_marks.size(); ++i) {
      float ms = 0.f;
      if (phase_marks[i].first >= 0 && cudaEventElapsedTime(&ms, phase_marks[i].second, phase_marks[i + 1].second) == cudaSuccess)
        phase_ms[phase_marks[i].first] += ms;
    }
    for (auto& m : phase_marks) cudaEventDestroy(m.second);
    phase_marks.clear();
  }
  void reset_stats() { for (auto& v : stats) v.store(0, std::memory_order_relaxed); if (profiling) for (auto& v : phase_ms) v = 0.f; }
  bool profiling = false;  // b200vs_set_profiling: time the dominant scan kernel with CUDA events
  virtual int export_nlist() const { return 1; }

  IndexBase(b200vs_type t, b200vs_metric m, int d, const b200vs_params& p);
  virtual ~IndexBase();
  void set_device() const { B200VS_CUDA(cudaSetDevice(device)); }
  bool ip_like() const { return metric == B200VS_IP || metric == B200VS_COSINE; }

  // rows in the index's row format (FP32, or packed bits on a binary index); a Flat or HNSW index needs no training
  virtual void train(int64_t n, const void* x) { (void)n; (void)x; }
  virtual bool is_trained() const { return true; }
  // the n of the train call that trained the index (IVF types); after a Load or a set_trained_state, the live count then
  int64_t train_rows = 0;
  // VectorIndex::NeedToRebuild (b200vs_need_rebuild): the reference plugin's rule for this type; callers hold rw shared
  virtual bool need_rebuild() const { return false; }
  // b200vs_rebuild_from[_range]: fill this empty, untrained index (rw and gpu_mu held, scratch reset, check_rebuild_pair
  // passed for every source) from the live rows with lo <= id <= hi of srcs in ascending id order, as a fresh train + add of
  // them would; the sources are held shared.  Returns the rows.
  virtual int64_t rebuild_from(const std::vector<IndexBase*>& srcs, int64_t lo, int64_t hi) {
    (void)srcs; (void)lo; (void)hi;
    fail(B200VS_EVECTOR_NOT_SUPPORT, "rebuild is not supported for this index type");
  }
  // this index's live rows with lo <= id <= hi as a rebuild source (sorted_live_rows).  Callers hold rw.
  virtual void live_rows(int64_t lo, int64_t hi, RebuildSource& out) {
    (void)lo; (void)hi; (void)out;
    fail(B200VS_EVECTOR_NOT_SUPPORT, "this index type has no row store to rebuild from");
  }
  // the ids of this index's live rows with lo <= id <= hi, appended to out in storage order (the refusals a sharded rebuild
  // agrees on before any rank's dst changes).  Callers hold rw.
  virtual void live_ids(int64_t lo, int64_t hi, std::vector<int64_t>& out) {
    RebuildSource p;
    live_rows(lo, hi, p);
    out.insert(out.end(), p.ids.begin(), p.ids.end());
  }
  // b200vs_brute_force_*: the types whose stored rows a brute-force scan reproduces (FLAT, IVF_FLAT, and HNSW under L2 / IP:
  // IVF_PQ keeps only codes, binary rows have no brute-force path, HNSW cosine rows carry NormalizeVectorForHnsw's bits)
  bool brute_force_served() const { return type == B200VS_FLAT || type == B200VS_IVF_FLAT || (type == B200VS_HNSW && metric != B200VS_COSINE); }
  // every row slot of a served index as one Flat view, on stream s with a lane held under the reader lock: the store's rows
  // and ids, or (where the store's ids do not say so) ids built per call in the lane's scratch, -1 for every tombstone,
  // unused slot or deleted node.  norms: the row norms the tile scan needs (HNSW computes them per call).  False when there
  // is nothing to scan (an empty or untrained index).
  virtual bool brute_force_rows(TcView& v, bool norms, cudaStream_t s) {
    (void)v; (void)norms; (void)s;
    fail(B200VS_EVECTOR_NOT_SUPPORT, "brute-force search over an index's rows is served for FLAT, IVF_FLAT and HNSW under L2 / IP");
  }
  virtual void set_state(const void* blob, size_t len) { (void)blob; (void)len; fail(B200VS_EVECTOR_NOT_SUPPORT, "no trained state for this index type"); }
  virtual int64_t get_state(void* blob, size_t cap) { (void)blob; (void)cap; return 0; }
  // THE write of rows into an index, under the writer hold.  Each type refuses the requests it cannot serve.
  virtual void add(const AddReq& r) = 0;
  // the refusals add(r) would give, decided from r's host ids and sizes before anything changes, so that every rank of a
  // collective add can agree on one status first (every type: a negative id; FLAT, BINARY_FLAT: a repeated id; HNSW:
  // max_elements, the batched plan).  Overrides begin with this one.
  virtual void check_add(const AddReq& r) { if (r.ids) check_ids_nonnegative(r.n, r.ids); }
  virtual int64_t remove(int64_t n, const int64_t* ids) = 0;
  virtual void clear() { fail(B200VS_EVECTOR_NOT_SUPPORT, "clear is only implemented for FLAT"); }  // drop every row, keep the buffers
  // THE read of an index, on stream s with the lane's scratch already reset: r's top-k or range search.  Each type refuses
  // the requests it cannot serve (a probe table without inverted lists, range on HNSW).
  virtual void search(const SearchReq& r, cudaStream_t s) = 0;
  // the coarse quantiser of the IVF types over centroid rows [c0, c1) (xq: query rows in the index's row format, FP32 or
  // packed bits): out_lists [nq, nprobe] global list ids (set semantics), and when out_score is set the ascending ranking
  // score of each (L2 distance | -ip | Hamming distance) in (score, list id) order
  virtual void coarse(int64_t nq, const void* xq, bool prepared, int nprobe, int c0, int c1, float* out_score, long long* out_lists,
                      cudaStream_t s) {
    (void)nq; (void)xq; (void)prepared; (void)nprobe; (void)c0; (void)c1; (void)out_score; (void)out_lists; (void)s;
    fail(B200VS_EVECTOR_NOT_SUPPORT, "coarse quantiser only exists for IVF_FLAT and IVF_PQ");
  }
  // ---- the building blocks of a list-sharded deployment (shard.cu); IVF_FLAT, IVF_PQ and BINARY_IVF_FLAT.  Row pointers
  // are in the index's row format: FP32 rows, or packed bits (dim / 8 bytes) on a binary index.
  // the refusals a search with k and sp's efsearch would meet after the first collective of a row-sharded search, decided
  // from the arguments and the index's parameters alone, so that every rank refuses alike before it (HNSW: efsearch outside
  // [0, 1024], as b200vs_search; the walk's shared memory)
  virtual void check_row_search(int k, const b200vs_search_params* sp) const { (void)k; (void)sp; }
  // nearest-centroid assignment of prepared rows (faiss quantizer->assign; the index's row format): out_lists_dev[n], on
  // stream s (a lane must be held)
  virtual void assign_lists_dev(int64_t n, const void* x_dev, long long* out_lists_dev, cudaStream_t s) {
    (void)n; (void)x_dev; (void)out_lists_dev; (void)s;
    fail(B200VS_EVECTOR_NOT_SUPPORT, "list assignment only exists for IVF_FLAT and IVF_PQ");
  }
  // pre-size every inverted list (rows_per_list[nlist]) in ONE arena allocation: bulk builds of large shards never
  // relocate a list or re-allocate the arena (a 77 GB shard cannot afford a 2x peak)
  virtual void reserve_lists(const int64_t* rows_per_list, int nlist) {
    (void)rows_per_list; (void)nlist;
    fail(B200VS_EVECTOR_NOT_SUPPORT, "list reservation only exists for IVF_FLAT and IVF_PQ");
  }
  virtual int nlist_now() const { return 1; }
  virtual int resolve_nprobe_api(const SearchCtx& sc) const { (void)sc; return 1; }
  // refusals of a search over a caller's probe table that depend only on nq, k and the trained state (IVF-PQ: the LUT + select pool
  // must fit one SM's shared memory; deep: the LUT alone, the deep key pass holds no select pool); a sharded search checks them on
  // every rank before its first collective
  virtual void check_probe_search(int64_t nq, int k, bool deep = false) const { (void)nq; (void)k; (void)deep; }
  // b200vs_debug_tc_scores: xq device (raw), outputs host [nq, count() + deleted_count()] and [nq]
  virtual void debug_tc_scores(int64_t nq, const float* xq, int arith, float* out_scores, float* out_eps, cudaStream_t s) {
    (void)nq; (void)xq; (void)arith; (void)out_scores; (void)out_eps; (void)s;
    fail(B200VS_EILLEGAL_PARAMETERS, "tensor-core score diagnostics only exist for FLAT");
  }

  // ---- binary indexes (B200VS_BINARY_FLAT / B200VS_BINARY_IVF_FLAT, binary.cu): rows are packed bits, dim / 8 bytes each.
  // The float entry points refuse a binary index, and the b200vs_*_binary ones a float index (api.cu).
  bool binary() const { return type == B200VS_BINARY_FLAT || type == B200VS_BINARY_IVF_FLAT; }
  size_t query_row_bytes() const { return binary() ? (size_t)dim / 8 : (size_t)dim * 4; }  // one host query row

  virtual void reconstruct(int64_t n, const int64_t* ids, float* out, uint8_t* found) {
    (void)n; (void)ids; (void)out; (void)found;
    fail(B200VS_EVECTOR_NOT_SUPPORT, "reconstruct is implemented for HNSW and FLAT");
  }
  virtual int sub_type() const { return (int)type; }
  virtual int64_t count() const = 0;
  virtual int64_t deleted_count() const { return 0; }
  virtual int64_t memory_size() const = 0;
  virtual void export_lists(int64_t* list_off, float* vectors, uint8_t* codes, int64_t* ids) = 0;
  virtual int64_t export_list(int list, int64_t cap, float* vectors, int64_t* ids) {
    (void)list; (void)cap; (void)vectors; (void)ids;
    fail(B200VS_EVECTOR_NOT_SUPPORT, "single-list export only exists for IVF_FLAT");
  }
  virtual void save(const std::string& path);
  virtual void load(const std::string& path);
  // b200vs_save_stage: into img, the bytes save(path) would write now.  The rows are packed on the device (pack_lists), and
  // the rest comes from the host bookkeeping.
  virtual void save_image(SnapshotImage& img);
  // export_lists' list offsets, ids and rows (in export_lists' host row format) of the live rows, gathered by one device pack
  // and brought back with one copy per buffer on the index stream.  out_ids and out_rows need no alignment.
  virtual void pack_lists(int64_t* list_off, void* out_ids, uint8_t* out_rows) {
    (void)list_off; (void)out_ids; (void)out_rows;
    fail(B200VS_EVECTOR_NOT_SUPPORT, "this index type has no device rows to pack");
  }

  // helpers shared by the index types
  // An AddReq's rows and ids on this device and its ids on the host, with the writer hold taken.  Host rows (row_bytes each)
  // and ids are uploaded to the scratch on the index stream, ids the caller did not give on the host are downloaded, and
  // device rows are copied to the scratch only when `own` asks for rows the add may change in place.  A negative id is
  // refused here, before the add changes anything.
  struct Staged {
    void* x = nullptr;  // the scratch copy, or the caller's device rows, which are only read
    const long long* ids_dev = nullptr;
    const int64_t* ids = nullptr;
    std::vector<int64_t> ids_buf;
  };
  void stage(const AddReq& r, size_t row_bytes, bool own, Staged& st);
  const float* prepare_queries(int64_t nq, const float* xq_dev, cudaStream_t s);  // cosine -> normalised copy
  const float* queries(const SearchReq& r, cudaStream_t s) { return r.prepared ? r.fq() : prepare_queries(r.nq, r.fq(), s); }
  // the refusal of a caller's probe table by a type without inverted lists to probe
  static void refuse_probes(const SearchReq& r) {
    if (r.probes) fail(B200VS_EVECTOR_NOT_SUPPORT, "probe-driven search only exists for IVF_FLAT and IVF_PQ");
  }
  void launch_count(int n = 1) { stats[0] += n; }
};

// Shared (reader) hold of an index's rw lock that composes: an operation made of several locked steps (Save = count, then
// trained state, then list export) takes it once at the top, the steps' own guards then see the hold and do not lock again
// (re-acquiring a std::shared_mutex in shared mode can dead-lock behind a queued writer, and releasing it between the steps
// lets an add grow the index past the buffers sized from the earlier count).
struct RwSharedGuard {
  static thread_local const IndexBase* tl_held;
  const IndexBase* prev;
  std::shared_lock<std::shared_mutex> lk;
  explicit RwSharedGuard(IndexBase* ix) : prev(tl_held) {
    if (tl_held != ix) { lk = std::shared_lock<std::shared_mutex>(ix->rw); tl_held = ix; }
  }
  ~RwSharedGuard() { tl_held = prev; }
  RwSharedGuard(const RwSharedGuard&) = delete;
  RwSharedGuard& operator=(const RwSharedGuard&) = delete;
};

// The writer prologue: rw exclusively, then gpu_mu, the index's device, every earlier search finished and the scratch reset
// on the index stream.  Every write of an index (add, remove, train, clear, reserve, trained state) runs under one.
struct WriteHold {
  std::unique_lock<std::shared_mutex> wl;
  std::lock_guard<std::mutex> gl;
  explicit WriteHold(IndexBase* ix) : wl(ix->rw), gl(ix->gpu_mu) {
    ix->set_device();
    ix->quiesce();
    ix->scratch.reset(ix->stream);
  }
};

// RAII: pick a lane for a search on stream `s` (nullptr = a lane-owned stream), lock it, make it the thread's scratch
struct LaneGuard {
  IndexBase* ix;
  Lane* lane;
  IndexBase* prev_owner;
  Lane* prev_lane;
  cudaStream_t stream;
  LaneGuard(IndexBase* ix_, cudaStream_t s);
  ~LaneGuard();
};

inline IndexBase* index_impl(b200vs_index* h) {
  if (!h || !h->impl) fail(B200VS_EILLEGAL_PARAMETERS, "null index handle");
  return h->impl;
}

IndexBase* make_flat(b200vs_metric m, int d, const b200vs_params& p);
IndexBase* make_ivf_flat(b200vs_metric m, int d, const b200vs_params& p);
IndexBase* make_ivf_pq(b200vs_metric m, int d, const b200vs_params& p);
IndexBase* make_hnsw(b200vs_metric m, int d, const b200vs_params& p);
// The live labels, in node order, of the graph in an HNSW state blob for the HNSW index ix, which stays untouched; refuses
// every blob that set_state refuses (hnsw.cu)
std::vector<int64_t> hnsw_state_labels(const IndexBase* ix, const void* blob, size_t len);
// IVF-PQ training in the two stages of its train (ivf_pq.cu), for the list-sharded trainer (shard.cu); ix must be an IVF_PQ
// index, whose lists and trained state stay untouched.  Coarse: k centroids of n raw rows.  State: the codebooks of the PQ
// rule on the n rows' residuals to the centroids cent [nlist, dim], returned with cent as a trained-state blob.
int ivf_pq_ksub(IndexBase* ix);
void ivf_pq_train_coarse(IndexBase* ix, int64_t n, const float* x, int k, std::vector<float>& cent);
void ivf_pq_train_state(IndexBase* ix, int64_t n, const float* x, const std::vector<float>& cent, std::vector<unsigned char>& blob);
// The same two stages for IVF_FLAT (index.cu); ix must be an IVF_FLAT index, which stays untouched.  Coarse: train's k
// centroids of n >= k rows: raw host rows, or (x_dev) prepared rows on ix's device, which are not normalised again
// (b200vs_rebuild_from's rule).  State: the trained-state blob of the centroids cent [nlist, dim].
void ivf_flat_train_coarse(IndexBase* ix, int64_t n, const float* x, bool x_dev, int k, std::vector<float>& cent);
void ivf_flat_train_state(IndexBase* ix, const std::vector<float>& cent, std::vector<unsigned char>& blob);
IndexBase* make_binary_flat(int d, const b200vs_params& p);
IndexBase* make_binary_ivf(int d, const b200vs_params& p);
// The same two stages for BINARY_IVF_FLAT (binary.cu); ix must be a BINARY_IVF_FLAT index, whose lists and trained state stay
// untouched.  Coarse: b200vs_train_binary's k packed centroids [k, dim / 8] of n >= k host packed rows x, or of n padded
// rows x_words [n, ceil(dim / 32)] on ix's device (x then null), whose sample is expanded to +-1 floats there.  State: the
// trained-state blob of the packed centroids cent [nlist, dim / 8].
void binary_ivf_train_coarse(IndexBase* ix, int64_t n, const uint8_t* x, const uint32_t* x_words, int k, std::vector<uint8_t>& cent);
void binary_ivf_train_state(IndexBase* ix, const std::vector<uint8_t>& cent, std::vector<unsigned char>& blob);

// ---- generic exact scan + select driver (scan_kernels.cuh) ----
struct ScanJob {
  bool l2 = true;
  bool hamming = false;  // binary rows: vecs / queries hold 32-bit words, d = words per row; l2 stays true (ascending)
  const float* vecs = nullptr;
  const long long* ids = nullptr;
  int d = 0;
  int mode = 0;
  long long n = 0;
  const long long* probes = nullptr;
  int nprobe = 0;
  const long long* list_off = nullptr;
  const int* list_len = nullptr;
  double avg_candidates = 0;  // expected candidates per query (sizing of nsplit)
  const SearchCtx* sc = nullptr;
  bool has_thr = false;
  float thr_raw = 0;  // range search: raw metric threshold (L2: dist < thr ; IP: ip > thr)
  bool dominant = false;  // the list scan of an IVF search: timed when profiling is on
};
// profiling helpers: distinct probed lists / rows of a probe table
void profile_probed(IndexBase* ix, const long long* probes, int64_t n_probes, int nlist, const int* list_len, cudaStream_t s);
struct ScopedKernelTimer {  // CUDA events on the launching stream; synchronises in the destructor
  IndexBase* ix; cudaStream_t s; cudaEvent_t e0 = nullptr, e1 = nullptr; bool on;
  ScopedKernelTimer(IndexBase* ix_, cudaStream_t s_, bool on_) : ix(ix_), s(s_), on(on_) {
    if (!on) return;
    B200VS_CUDA(cudaEventCreate(&e0)); B200VS_CUDA(cudaEventCreate(&e1)); B200VS_CUDA(cudaEventRecord(e0, s));
  }
  void stop() {
    if (!on || !e0) return;
    cudaEventRecord(e1, s); cudaEventSynchronize(e1);
    float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
    ix->stats[3] += (int64_t)(ms * 1e6);
    cudaEventDestroy(e0); cudaEventDestroy(e1); e0 = e1 = nullptr;
  }
  ~ScopedKernelTimer() { stop(); }
};
// results: out_dist (API), out_raw (raw metric), out_ids, out_counts — any but out_ids may be null
void run_scan(IndexBase* ix, const ScanJob& job, int64_t nq, const float* queries, int k, float* out_dist,
              float* out_raw, long long* out_ids, int* out_counts, cudaStream_t s);

// ---- deep top-k (deep_select.cu): exact top-k for k up to kDeepMaxK, past what the shared-memory select holds ----
constexpr int kDeepMaxK = B200VS_DEEP_MAX_K;
// A deep search's candidate space.  mode 0: candidate i of query q is row q * row_stride + i of [0, n) (row_stride 0: one
// index for every query); mode 1: the probe-prefix positions of the lists probes[q] (the exact scan's map_row rule).
struct DeepJob {
  bool l2 = true;         // the key order of the scan: L2 / Hamming distance, or -ip
  bool api_keys = false;  // the keys are f2ord(API distance) (a merge of result lists): emit the key's own float
  int mode = 0;
  long long n = 0, row_stride = 0;
  const long long* ids = nullptr;
  const long long* probes = nullptr;
  int nprobe = 0;
  const long long* list_off = nullptr;
  const int* list_len = nullptr;
};
// the key pass of queries [q0, q0 + nqc): fills o's keys, eligibility and counts on stream s
using DeepKeyPass = std::function<void(int64_t q0, int nqc, const DeepKeys& o, cudaStream_t s)>;
// top-k of nq queries: od [nq, k] (the API distance, or the raw metric value when raw; may be null), oi [nq, k], -1 padded
void run_deep(IndexBase* ix, const DeepJob& job, int64_t nq, int k, float* od, bool raw, long long* oi, const DeepKeyPass& pass,
              cudaStream_t s);
// merge_api_kernel's merge through run_deep: the top k of each query's n API-distance slots cat_d / cat_i [nq, n] (id < 0:
// empty), ordered by (distance, id), into od / oi [nq, k]
void run_deep_merge_api(IndexBase* ix, int64_t nq, int k, int n, const float* cat_d, const long long* cat_i, float* od, long long* oi,
                        cudaStream_t s);
// whether the exact scan's shared-memory select serves top-k k over d-float rows and nseg probed lists (run_scan, and the
// merge kernels over the same pool)
bool exact_select_fits(int d, int nseg, int k);
// run_deep over the exact scan of job (scan_key_kernel)
void run_scan_deep(IndexBase* ix, const ScanJob& job, int64_t nq, const float* queries, int k, float* od, bool raw, long long* oi,
                   cudaStream_t s);

// b200vs_scan_range_push: append the hits of one tile [n, d] to each query's running list in row order (range_append_kernel).
// thr_raw is the raw threshold (L2: dist < thr; IP: ip > thr); counts[nq] persists across calls.  rows (nullable): the walk's
// i-th row is vecs row rows[i] with id ids[i] (b200vs_brute_force_range_search's gathered list), else row i.
void launch_range_append(bool l2, const float* vecs, const long long* ids, const long long* rows, int64_t n, int d, int64_t nq,
                         const float* queries, const SearchCtx& sc, float thr_raw, int max_results, float* out_dist,
                         long long* out_ids, int* counts, cudaStream_t s);
void launch_normalize_faiss(float* x, int64_t n, int d, cudaStream_t s);
void launch_normalize_hnsw(const float* x, float* out, int64_t n, int d, cudaStream_t s);
void launch_scatter_rows(const float* src, const long long* src_ids, const long long* slots, int64_t n, int d,
                         float* vecs, long long* ids, float* norms, float* row_norms, cudaStream_t s);
void launch_move_rows(const float* svecs, const long long* sids, const float* snorms, const long long* src_rows,
                      const long long* dst_rows, int64_t n, int d, float* dvecs, long long* dids, float* dnorms,
                      cudaStream_t s);
void launch_set_ids(long long* ids, const long long* slots, int64_t n, long long value, cudaStream_t s);
void launch_iota(long long* p, int64_t n, cudaStream_t s);
// out[r] = ids[r] for the rows r in [off[l], off[l] + len[l]) of some list l < nlist, -1 for every other r < rows
// (brute_force.cu)
void launch_list_ids(const long long* ids, const long long* off, const int* len, int nlist, int64_t rows, long long* out,
                     cudaStream_t s);
// out[i] = deleted[i] ? -1 : labels[i] for the n nodes of an HNSW device mirror (brute_force.cu)
void launch_node_ids(const long long* labels, const unsigned char* deleted, int64_t n, long long* out, cudaStream_t s);
void launch_negate(float* p, int64_t n, cudaStream_t s);
// out[i*nr + j] = L2 ? ||a_i - b_j||^2 : 1 - <a_i, b_j>, reference summation order (VectorCalcDistance)
void launch_pair_distance(bool l2, const float* a, int64_t nl, const float* b, int64_t nr, int d, float* out, cudaStream_t s);
// out[i*nr + j] = popcount(a_i XOR b_j) over w-word zero-padded binary rows (b200vs_calc_distance_binary)
void launch_pair_hamming(const uint32_t* a, int64_t nl, const uint32_t* b, int64_t nr, int w, float* out, cudaStream_t s);
// packed binary rows [n, nbytes] -> zero-padded 32-bit words [n, ceil(nbytes / 4)] (binary.cu)
void launch_pad_rows(const uint8_t* src, int64_t n, int nbytes, uint32_t* dst, cudaStream_t s);
void hnsw_build_scratch_limit(IndexBase* ix, int64_t bytes);  // b200vs_debug_hnsw_build_scratch_limit
void launch_merge_api(int nparts, int64_t nq, int k, const float* pd, const long long* pi, float* od, long long* oi,
                      cudaStream_t s);

}  // namespace b200vs
