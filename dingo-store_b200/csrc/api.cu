// api.cu — extern "C" entry points of libb200vs.so (declared in include/b200vs.h).
// No exception leaves this file: every entry point maps failures to a b200vs_status
// (reference convention: butil::Status codes, never exceptions across the plugin virtual;
// src/vector/vector_index_flat.cc:313-315, src/handler/raft_apply_handler.cc:1311-1325).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "index.h"
#include "ivf_common.h"

using namespace b200vs;

// b200vs_rebuild_from[_range]: fill dst from the live rows with lo <= id <= hi of srcs (distinct, dst not among them).  The
// sources are held under their reader locks and dst under its writer hold, taken in one order, by address, so two calls over
// overlapping sources (a split's child and parent rebuilding from the parent's index at once) cannot deadlock.  flat_ok:
// FLAT and BINARY_FLAT are served.
int64_t b200vs::rebuild_range(IndexBase* dst, const std::vector<IndexBase*>& srcs, int64_t lo, int64_t hi, bool flat_ok) {
  std::vector<IndexBase*> order(srcs);
  order.push_back(dst);
  std::sort(order.begin(), order.end(), std::less<IndexBase*>());
  std::vector<std::shared_lock<std::shared_mutex>> reads;
  std::unique_ptr<WriteHold> hold;
  for (IndexBase* ix : order) {
    if (ix == dst) hold.reset(new WriteHold(dst));
    else reads.emplace_back(ix->rw);
  }
  for (IndexBase* src : srcs) check_rebuild_pair(*dst, *src);
  if (!flat_ok && (dst->type == B200VS_FLAT || dst->type == B200VS_BINARY_FLAT))
    fail(B200VS_EVECTOR_NOT_SUPPORT, "a Flat index never needs a rebuild");  // vector_index_flat.h:111
  return dst->rebuild_from(srcs, lo, hi);
}

namespace {

IndexBase* get(b200vs_index* h) { return index_impl(h); }

// the float entry points (train / add / search / range search) on a binary index, and the binary ones on a float index
void check_row_type(IndexBase* ix, bool binary_call) {
  if (ix->binary() != binary_call)
    fail(B200VS_EILLEGAL_PARAMETERS, binary_call ? "binary entry point on a float index" : "float entry point on a binary index");
}

// The list building blocks take FP32 rows: a binary index refuses them as the index layer did before it served binary
// shards (b200vs_shard_*_binary reach those hooks with packed rows)
void refuse_binary_rows(IndexBase* ix, const char* what) {
  if (ix->binary()) fail(B200VS_EVECTOR_NOT_SUPPORT, std::string(what) + " only exists for IVF_FLAT and IVF_PQ");
}

void check_search_args(IndexBase* ix, int64_t nq, const void* xq, const b200vs_search_params* sp) {
  if (nq <= 0 || !xq) fail(B200VS_EILLEGAL_PARAMETERS, "vector_with_ids is empty");  // flat.cc:208-210
  if (ix->type == B200VS_HNSW && sp && (sp->efsearch < 0 || sp->efsearch > 1024))
    fail(B200VS_EILLEGAL_PARAMETERS, "efsearch is illegal, " + std::to_string(sp->efsearch) + ", must between 0 and 1024");  // hnsw.cc:332-336
}

// The prologue and epilogue of every read of one index: the shared lock, the device, a lane on `stream` (null: the lane's
// own stream), fresh stats and the resolved search parameters, then body(sc, s) on the lane's stream, the profiling phases,
// and for a null stream the wait for the results.
template <class Body>
void index_read(IndexBase* ix, void* stream, const b200vs_search_params* sp, Body body) {
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  ix->set_device();
  LaneGuard lane(ix, (cudaStream_t)stream);
  const cudaStream_t s = lane.stream;
  ix->reset_stats();
  const SearchCtx sc = make_ctx(ix, sp, s);
  body(sc, s);
  ix->phases_finish(s);
  if (!stream) B200VS_CUDA(cudaStreamSynchronize(s));  // NULL stream: library-owned stream, results ready on return
}

// One host-pointer read: nq query rows of query_row_bytes() (floats, or packed bits on a binary index) go up, the index
// answers into scratch, and the results come down into out_dist / out_ids [nq, k] (and, for a range search, out_counts
// [nq]).  A NaN radius admits no row of a float index: empty results, nothing launched (DESIGN.md 4.6); a binary index
// refuses it.  xq / outputs may be pinned staging (coalesced batches) or caller memory.
// brute: every stored row (b200vs_brute_force_*) in place of the index's own search.
void host_read(IndexBase* ix, int64_t nq, const void* xq, int k, const b200vs_search_params* sp, float* out_dist, int64_t* out_ids,
               bool range = false, float radius = 0.f, int32_t* out_counts = nullptr, bool deep = false, bool brute = false) {
  index_read(ix, nullptr, sp, [&](const SearchCtx& sc, cudaStream_t s) {
    const size_t nk = (size_t)nq * k;
    if (brute && !ix->brute_force_served())  // before anything is launched, with the stats already cleared
      fail(B200VS_EVECTOR_NOT_SUPPORT, "brute-force search over an index's rows is served for FLAT, IVF_FLAT and HNSW under L2 / IP");
    if (range && std::isnan(radius) && !ix->binary()) {
      std::fill_n(out_dist, nk, 0.0F);
      std::fill_n(out_ids, nk, (int64_t)-1);
      std::fill_n(out_counts, (size_t)nq, 0);
      return;
    }
    const size_t qbytes = (size_t)nq * ix->query_row_bytes();
    SearchReq r;
    r.nq = nq; r.k = k; r.range = range; r.radius = radius; r.sc = &sc; r.deep = deep;
    void* dq = ix->scratch.alloc<unsigned char>(qbytes);
    r.xq = dq;
    r.od = ix->scratch.alloc<float>(nk);
    r.oi = ix->scratch.alloc<long long>(nk);
    if (range) r.oc = ix->scratch.alloc<int>((size_t)nq);
    B200VS_CUDA(cudaMemcpyAsync(dq, xq, qbytes, cudaMemcpyHostToDevice, s));
    if (brute) brute_force(ix, r, s);
    else ix->search(r, s);
    ix->phases_finish(s);  // the phases end before the copies back
    B200VS_CUDA(cudaMemcpyAsync(out_dist, r.od, nk * 4, cudaMemcpyDeviceToHost, s));
    B200VS_CUDA(cudaMemcpyAsync(out_ids, r.oi, nk * 8, cudaMemcpyDeviceToHost, s));
    if (range) B200VS_CUDA(cudaMemcpyAsync(out_counts, r.oc, (size_t)nq * 4, cudaMemcpyDeviceToHost, s));
  });
}

// b200vs_search_device / b200vs_search_binary_device
int search_device(b200vs_index* h, int64_t nq, const void* xq_dev, int k, const b200vs_search_params* sp, float* out_dist_dev,
                  int64_t* out_ids_dev, void* stream, bool binary) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    check_row_type(ix, binary);
    check_search_args(ix, nq, xq_dev, sp);
    if (k <= 0) return B200VS_OK;  // "topk <= 0 -> OK", flat.cc:212
    if (!out_ids_dev) fail(B200VS_EILLEGAL_PARAMETERS, "null output");
    index_read(ix, stream, sp, [&](const SearchCtx& sc, cudaStream_t s) {
      SearchReq r;
      r.nq = nq; r.xq = xq_dev; r.k = k; r.sc = &sc; r.od = out_dist_dev; r.oi = (long long*)out_ids_dev;
      ix->search(r, s);
    });
    return B200VS_OK;
  });
}

// b200vs_range_search / b200vs_range_search_binary
int range_search(b200vs_index* h, int64_t nq, const void* xq, float radius, int max_results, const b200vs_search_params* sp,
                 float* out_dist, int64_t* out_ids, int32_t* out_counts, bool binary) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    check_row_type(ix, binary);
    check_search_args(ix, nq, xq, sp);
    if (ix->type == B200VS_HNSW) fail(B200VS_EVECTOR_NOT_SUPPORT, "RangeSearch not support in Hnsw!!!");  // hnsw.cc:487-493
    if (max_results <= 0 || !out_ids || !out_dist || !out_counts) fail(B200VS_EILLEGAL_PARAMETERS, "bad range-search outputs");
    host_read(ix, nq, xq, max_results, sp, out_dist, out_ids, true, radius, out_counts);
    return B200VS_OK;
  });
}

// b200vs_brute_force_search / b200vs_brute_force_range_search: the arguments' checks and statuses of b200vs_scan_begin /
// b200vs_scan_range_begin; host_read refuses the types whose rows the scan cannot reproduce
int host_brute_force(b200vs_index* h, int64_t nq, const float* xq, int k, bool range, float radius, const b200vs_search_params* sp,
                     float* out_dist, int64_t* out_ids, int32_t* out_counts) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    if (nq <= 0 || !xq) fail(B200VS_EILLEGAL_PARAMETERS, "vector_with_ids is empty");
    if (range) {
      if (k <= 0) fail(B200VS_EILLEGAL_PARAMETERS, "max_results must be > 0");
      if (!out_counts) fail(B200VS_EILLEGAL_PARAMETERS, "null output");
    } else {
      if (k <= 0) return B200VS_OK;
      if (k > kDeepMaxK) fail(B200VS_EILLEGAL_PARAMETERS, "topk above " + std::to_string(kDeepMaxK));
    }
    if (!out_ids || !out_dist) fail(B200VS_EILLEGAL_PARAMETERS, "null output");
    // the top-k of b200vs_scan_*: the deep path past the exact scan's shared-memory select
    const bool deep = !range && !exact_select_fits(ix->dim, 1, k);
    host_read(ix, nq, xq, k, sp, out_dist, out_ids, range, radius, out_counts, deep, true);
    return B200VS_OK;
  });
}

}  // namespace

extern "C" {

int b200vs_brute_force_search(b200vs_index* h, int64_t nq, const float* xq, int32_t k, const b200vs_search_params* sp, float* out_dist,
                              int64_t* out_ids) {
  return host_brute_force(h, nq, xq, k, false, 0.f, sp, out_dist, out_ids, nullptr);
}

int b200vs_brute_force_range_search(b200vs_index* h, int64_t nq, const float* xq, float radius, int32_t max_results,
                                    const b200vs_search_params* sp, float* out_dist, int64_t* out_ids, int32_t* out_counts) {
  return host_brute_force(h, nq, xq, max_results, true, radius, sp, out_dist, out_ids, out_counts);
}

int b200vs_create(b200vs_type type, b200vs_metric metric, int32_t dim, const b200vs_params* params, b200vs_index** out) {
  return guarded([&]() -> int {
    if (!out) fail(B200VS_EILLEGAL_PARAMETERS, "out is null");
    *out = nullptr;
    if (dim <= 0) fail(B200VS_EILLEGAL_PARAMETERS, "dimension must be > 0");
    const bool binary = type == B200VS_BINARY_FLAT || type == B200VS_BINARY_IVF_FLAT;
    if (binary) {  // vector_index_utils.cc:1075-1140: HAMMING only, dimension in bits, dim % 8 == 0, dim <= kVectorMaxDimension
      if (metric != B200VS_HAMMING) fail(B200VS_EILLEGAL_PARAMETERS, "binary indexes support only METRIC_TYPE_HAMMING");
      if (dim % 8 != 0 || dim > 32768) fail(B200VS_EILLEGAL_PARAMETERS, "binary dimension must be a multiple of 8 in (0, 32768]");
    } else if (metric != B200VS_L2 && metric != B200VS_IP && metric != B200VS_COSINE) {
      fail(B200VS_EILLEGAL_PARAMETERS, "unsupported metric type");
    }
    b200vs_params p;
    memset(&p, 0, sizeof(p));
    if (params) p = *params;
    int ndev = 0;
    B200VS_CUDA(cudaGetDeviceCount(&ndev));
    if (p.device < 0 || p.device >= ndev) fail(B200VS_EILLEGAL_PARAMETERS, "bad CUDA device ordinal");
    IndexBase* impl = nullptr;
    switch (type) {
      case B200VS_FLAT: impl = make_flat(metric, dim, p); break;
      case B200VS_IVF_FLAT: impl = make_ivf_flat(metric, dim, p); break;
      case B200VS_IVF_PQ: impl = make_ivf_pq(metric, dim, p); break;
      case B200VS_HNSW: impl = make_hnsw(metric, dim, p); break;
      case B200VS_BINARY_FLAT: impl = make_binary_flat(dim, p); break;
      case B200VS_BINARY_IVF_FLAT: impl = make_binary_ivf(dim, p); break;
      default: fail(B200VS_EILLEGAL_PARAMETERS, "unknown index type");
    }
    *out = new b200vs_index{impl};
    return B200VS_OK;
  });
}

void b200vs_destroy(b200vs_index* h) {
  if (!h) return;
  try { delete h->impl; } catch (...) {}
  delete h;
}

int b200vs_train(b200vs_index* h, int64_t n, const float* x) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    check_row_type(ix, false);
    if (n <= 0 || !x) fail(B200VS_EILLEGAL_PARAMETERS, "data size invalid");  // ivf_flat.cc:646-649
    ix->train(n, x);
    return B200VS_OK;
  });
}

int b200vs_set_trained_state(b200vs_index* h, const void* blob, size_t len) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    if (!blob) fail(B200VS_EILLEGAL_PARAMETERS, "null blob");
    int64_t live = 0;
    { std::shared_lock<std::shared_mutex> rl(ix->rw); live = ix->count(); }
    ix->set_state(blob, len);
    std::unique_lock<std::shared_mutex> wl(ix->rw);
    ix->train_rows = live;  // the rule's training size: the live count at this call, as a Load sets it
    return B200VS_OK;
  });
}

int64_t b200vs_get_trained_state(b200vs_index* h, void* blob, size_t cap) {
  int64_t r = 0;
  int rc = guarded([&]() -> int { r = get(h)->get_state(blob, cap); return B200VS_OK; });
  return rc == B200VS_OK ? r : -(int64_t)rc;
}

int b200vs_add_with_ids(b200vs_index* h, int64_t n, const float* x, const int64_t* ids, int upsert) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    check_row_type(ix, false);
    if (n <= 0 || !x || !ids) fail(B200VS_EILLEGAL_PARAMETERS, "vector_with_ids is empty");  // flat.cc:123-125
    ix->add(AddReq::host(n, x, ids, upsert != 0));
    return B200VS_OK;
  });
}

int b200vs_hnsw_add_batched(b200vs_index* h, int64_t n, const float* x, const int64_t* ids, int32_t batch) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    if (ix->type != B200VS_HNSW) fail(B200VS_EILLEGAL_PARAMETERS, "batched HNSW construction needs an HNSW index");
    if (n <= 0 || !x || !ids) fail(B200VS_EILLEGAL_PARAMETERS, "vector_with_ids is empty");
    AddReq r = AddReq::host(n, x, ids);
    r.batched = true;
    r.batch = batch;
    ix->add(r);
    return B200VS_OK;
  });
}

int b200vs_debug_hnsw_build_scratch_limit(b200vs_index* h, int64_t bytes) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    if (ix->type != B200VS_HNSW || bytes < 0) fail(B200VS_EILLEGAL_PARAMETERS, "scratch limit needs an HNSW index and bytes >= 0");
    hnsw_build_scratch_limit(ix, bytes);
    return B200VS_OK;
  });
}

int b200vs_add_with_ids_device(b200vs_index* h, int64_t n, const float* x_dev, const int64_t* ids_dev, const int64_t* lists_dev, int upsert) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    if (n <= 0 || !x_dev || !ids_dev) fail(B200VS_EILLEGAL_PARAMETERS, "vector_with_ids is empty");
    if (ix->type != B200VS_IVF_FLAT && ix->type != B200VS_IVF_PQ)
      fail(B200VS_EVECTOR_NOT_SUPPORT, "device-pointer add only exists for IVF_FLAT and IVF_PQ");
    ix->add(AddReq::device(n, x_dev, (const long long*)ids_dev, (const long long*)lists_dev, upsert != 0));
    return B200VS_OK;
  });
}

int b200vs_assign_device(b200vs_index* h, int64_t n, const float* x_dev, int64_t* out_lists_dev) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    if (n <= 0 || !x_dev || !out_lists_dev) fail(B200VS_EILLEGAL_PARAMETERS, "bad assign arguments");
    refuse_binary_rows(ix, "list assignment");
    std::shared_lock<std::shared_mutex> rl(ix->rw);
    ix->set_device();
    LaneGuard lane(ix, nullptr);
    const float* q = ix->prepare_queries(n, x_dev, lane.stream);
    ix->assign_lists_dev(n, q, (long long*)out_lists_dev, lane.stream);
    B200VS_CUDA(cudaStreamSynchronize(lane.stream));
    return B200VS_OK;
  });
}

int b200vs_reserve_lists(b200vs_index* h, const int64_t* rows_per_list, int32_t nlist) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    if (!rows_per_list || nlist <= 0) fail(B200VS_EILLEGAL_PARAMETERS, "bad reserve arguments");
    ix->reserve_lists(rows_per_list, nlist);
    return B200VS_OK;
  });
}

int b200vs_remove_ids(b200vs_index* h, int64_t n, const int64_t* ids, int64_t* n_removed) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    if (n_removed) *n_removed = 0;
    if (n <= 0) return B200VS_OK;  // "delete_ids.empty() -> OK", flat.cc:172-174
    if (!ids) fail(B200VS_EILLEGAL_PARAMETERS, "null ids");
    const int64_t r = ix->remove(n, ids);
    if (n_removed) *n_removed = r < 0 ? 0 : r;
    // IVF types: "remove not found vector id" -> EVECTOR_INVALID (ivf_flat.cc:180-184); untrained -> OK (r == -1)
    if (r == 0 && (ix->type == B200VS_IVF_FLAT || ix->type == B200VS_IVF_PQ || ix->type == B200VS_BINARY_IVF_FLAT))
      fail(B200VS_EVECTOR_INVALID, "remove not found vector id");
    return B200VS_OK;
  });
}

int b200vs_search_device(b200vs_index* h, int64_t nq, const float* xq_dev, int32_t k, const b200vs_search_params* sp,
                         float* out_dist_dev, int64_t* out_ids_dev, void* stream) {
  return search_device(h, nq, xq_dev, k, sp, out_dist_dev, out_ids_dev, stream, false);
}

int b200vs_coarse_device(b200vs_index* h, int64_t nq, const float* xq_dev, int32_t nprobe, int32_t list_begin, int32_t list_end,
                         float* out_score_dev, int64_t* out_lists_dev, void* stream) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    if (nq <= 0 || !xq_dev || !out_score_dev || !out_lists_dev) fail(B200VS_EILLEGAL_PARAMETERS, "bad coarse arguments");
    refuse_binary_rows(ix, "coarse quantiser");
    index_read(ix, stream, nullptr, [&](const SearchCtx&, cudaStream_t s) {
      ix->coarse(nq, xq_dev, false, nprobe, list_begin, list_end, out_score_dev, (long long*)out_lists_dev, s);
    });
    return B200VS_OK;
  });
}

int b200vs_search_probes_device(b200vs_index* h, int64_t nq, const float* xq_dev, int32_t k, const int64_t* probes_dev, int32_t nprobe,
                                const b200vs_search_params* sp, float* out_dist_dev, int64_t* out_ids_dev, void* stream) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    check_search_args(ix, nq, xq_dev, sp);
    if (k <= 0) return B200VS_OK;
    if (!probes_dev || nprobe <= 0 || !out_ids_dev) fail(B200VS_EILLEGAL_PARAMETERS, "bad probe arguments");
    refuse_binary_rows(ix, "probe-driven search");
    index_read(ix, stream, sp, [&](const SearchCtx& sc, cudaStream_t s) {
      SearchReq r;
      r.nq = nq; r.xq = xq_dev; r.probes = (const long long*)probes_dev; r.nprobe = nprobe; r.k = k; r.sc = &sc;
      r.od = out_dist_dev; r.oi = (long long*)out_ids_dev;
      ix->search(r, s);
    });
    return B200VS_OK;
  });
}

int b200vs_debug_tc_scores(b200vs_index* h, int64_t nq, const float* xq, int32_t split, float* out_scores, float* out_eps) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    if (ix->binary()) fail(B200VS_EVECTOR_NOT_SUPPORT, "binary indexes have no tensor-core scores");
    if (ix->type != B200VS_FLAT) fail(B200VS_EILLEGAL_PARAMETERS, "tensor-core score diagnostics only exist for FLAT");
    if (ix->dim % 4 != 0 || ix->dim < 32) fail(B200VS_EILLEGAL_PARAMETERS, "the tile kernel needs dim % 4 == 0 and dim >= 32");
    if (nq <= 0 || !xq || !out_scores || !out_eps) fail(B200VS_EILLEGAL_PARAMETERS, "bad diagnostic arguments");
    if (split < 0 || split > 4) fail(B200VS_EILLEGAL_PARAMETERS, "split must be 0, 1, 2, 3 or 4");
    if ((split == 2 || split == 4) && ix->dim % 8 != 0) fail(B200VS_EILLEGAL_PARAMETERS, "the FP16 arithmetic needs dim % 8 == 0");
    index_read(ix, nullptr, nullptr, [&](const SearchCtx&, cudaStream_t s) {
      float* dq = ix->scratch.alloc<float>((size_t)nq * ix->dim);
      B200VS_CUDA(cudaMemcpyAsync(dq, xq, (size_t)nq * ix->dim * 4, cudaMemcpyHostToDevice, s));
      ix->debug_tc_scores(nq, dq, split, out_scores, out_eps, s);
    });
    return B200VS_OK;
  });
}

}  // extern "C"

namespace {

bool coalesce_compatible(const CoalesceReq& a, const CoalesceReq& b) {
  return a.k == b.k && a.sp.nprobe == b.sp.nprobe && a.sp.efsearch == b.sp.efsearch && a.sp.exact_only == b.sp.exact_only &&
         a.sp.has_range == b.sp.has_range && (!a.sp.has_range || (a.sp.range_min == b.sp.range_min && a.sp.range_max == b.sp.range_max));
}

constexpr int64_t kCoalesceMaxReq = 64;     // requests at most this large join a shared batch
constexpr int64_t kCoalesceMaxBatch = 4096; // queries per shared batch (the service limit, index_service.cc:50)

// the leader's work: one batch for all requests in `batch` (>= 2 of them, compatible)
void run_coalesced(IndexBase* ix, std::vector<CoalesceReq*>& batch) {
  int64_t total = 0;
  for (auto* r : batch) total += r->nq;
  const int k = batch[0]->k;
  const size_t row = ix->query_row_bytes();
  // pinned staging owned by the calling (leader) thread: queries in, results out (one H2D, one D2H of each kind)
  const size_t qbytes = (size_t)total * row, dbytes = (size_t)total * k * 4, ibytes = (size_t)total * k * 8;
  const size_t need = qbytes + dbytes + ibytes + 64;
  static thread_local void* pin = nullptr;
  static thread_local size_t pin_cap = 0;
  if (pin_cap < need) {
    ix->set_device();
    if (pin) cudaFreeHost(pin);
    pin = nullptr; pin_cap = 0;
    B200VS_CUDA(cudaHostAlloc(&pin, need * 2, cudaHostAllocPortable));  // portable: the calling thread may serve indexes on several devices
    pin_cap = need * 2;
  }
  char* hq = reinterpret_cast<char*>(pin);
  float* hd = reinterpret_cast<float*>(hq + ((qbytes + 15) & ~(size_t)15));
  int64_t* hi = reinterpret_cast<int64_t*>(reinterpret_cast<char*>(hd) + ((dbytes + 15) & ~(size_t)15));
  int64_t off = 0;
  for (auto* r : batch) { memcpy(hq + (size_t)off * row, r->xq, (size_t)r->nq * row); off += r->nq; }
  host_read(ix, total, hq, k, &batch[0]->sp, hd, hi);
  off = 0;
  for (auto* r : batch) {
    memcpy(r->out_dist, hd + (size_t)off * k, (size_t)r->nq * k * 4);
    memcpy(r->out_ids, hi + (size_t)off * k, (size_t)r->nq * k * 8);
    off += r->nq;
  }
}

int coalesced_search(IndexBase* ix, int64_t nq, const void* xq, int k, const b200vs_search_params* sp, float* out_dist, int64_t* out_ids) {
  Coalescer& C = ix->coalescer;
  CoalesceReq me;
  me.nq = nq; me.xq = xq; me.k = k; me.out_dist = out_dist; me.out_ids = out_ids;
  if (sp) me.sp = *sp;
  std::unique_lock<std::mutex> lk(C.mu);
  C.pending.push_back(&me);
  while (!me.done) {
    if (C.busy) { C.cv.wait(lk); continue; }
    // become the leader: everything compatible with the oldest pending request, in arrival order
    C.busy = true;
    std::vector<CoalesceReq*> batch, rest;
    int64_t total = 0;
    for (auto* r : C.pending) {
      if ((batch.empty() || coalesce_compatible(*batch[0], *r)) && total + r->nq <= kCoalesceMaxBatch) { batch.push_back(r); total += r->nq; }
      else rest.push_back(r);
    }
    C.pending.swap(rest);
    lk.unlock();
    int rc = B200VS_OK;
    std::string err;
    try {
      if (batch.size() == 1) host_read(ix, batch[0]->nq, batch[0]->xq, batch[0]->k, &batch[0]->sp, batch[0]->out_dist, batch[0]->out_ids);
      else run_coalesced(ix, batch);
    } catch (const StatusError& e) { rc = e.code; err = e.msg; }
    catch (const std::exception& e) { rc = B200VS_EINTERNAL; err = e.what(); }
    catch (...) { rc = B200VS_EINTERNAL; err = "unknown error"; }
    C.batches.fetch_add(1);
    C.requests.fetch_add((int64_t)batch.size());
    lk.lock();
    for (auto* r : batch) { r->rc = rc; r->err = err; r->done = true; }
    C.busy = false;
    C.cv.notify_all();
  }
  lk.unlock();
  if (me.rc != B200VS_OK) g_last_error = me.err;
  return me.rc;
}

// b200vs_search / b200vs_search_binary: small filter-free requests share batches with concurrent callers (the reference
// issues one query per pool task)
int host_search(b200vs_index* h, int64_t nq, const void* xq, int k, const b200vs_search_params* sp, float* out_dist, int64_t* out_ids,
                bool binary) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    check_row_type(ix, binary);
    check_search_args(ix, nq, xq, sp);
    if (k <= 0) return B200VS_OK;
    if (!out_ids || !out_dist) fail(B200VS_EILLEGAL_PARAMETERS, "null output");
    if (nq <= kCoalesceMaxReq && ix->coalescer.enabled.load() && !(sp && sp->sorted_ids) && !ix->profiling)
      return coalesced_search(ix, nq, xq, k, sp, out_dist, out_ids);
    host_read(ix, nq, xq, k, sp, out_dist, out_ids);
    return B200VS_OK;
  });
}

// b200vs_search_deep / b200vs_search_binary_deep: the deep path for any k up to kDeepMaxK; never coalesced
int host_search_deep(b200vs_index* h, int64_t nq, const void* xq, int k, const b200vs_search_params* sp, float* out_dist,
                     int64_t* out_ids, bool binary) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    check_row_type(ix, binary);
    check_search_args(ix, nq, xq, sp);
    if (k <= 0) return B200VS_OK;
    if (k > kDeepMaxK) fail(B200VS_EILLEGAL_PARAMETERS, "topk above " + std::to_string(kDeepMaxK));
    if (ix->type == B200VS_HNSW) fail(B200VS_EVECTOR_NOT_SUPPORT, "deep top-k is not implemented for HNSW");
    if (!out_ids || !out_dist) fail(B200VS_EILLEGAL_PARAMETERS, "null output");
    host_read(ix, nq, xq, k, sp, out_dist, out_ids, false, 0.f, nullptr, true);
    return B200VS_OK;
  });
}

}  // namespace

extern "C" {

int b200vs_search_deep(b200vs_index* h, int64_t nq, const float* xq, int32_t k, const b200vs_search_params* sp, float* out_dist,
                       int64_t* out_ids) {
  return host_search_deep(h, nq, xq, k, sp, out_dist, out_ids, false);
}

int b200vs_search_binary_deep(b200vs_index* h, int64_t nq, const uint8_t* xq, int32_t k, const b200vs_search_params* sp,
                              float* out_dist, int64_t* out_ids) {
  return host_search_deep(h, nq, xq, k, sp, out_dist, out_ids, true);
}

int b200vs_search(b200vs_index* h, int64_t nq, const float* xq, int32_t k, const b200vs_search_params* sp, float* out_dist,
                  int64_t* out_ids) {
  return host_search(h, nq, xq, k, sp, out_dist, out_ids, false);
}

/* Request coalescing of b200vs_search and b200vs_search_binary (on by default): concurrent host-pointer calls of <= 64
 * queries without id-list filters are merged into shared batches.  stats (nullable): [0] batches run, [1] requests served
 * through them. */
int b200vs_set_coalescing(b200vs_index* h, int on, int64_t stats[2]) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    if (on >= 0) ix->coalescer.enabled.store(on ? 1 : 0);
    if (stats) { stats[0] = ix->coalescer.batches.load(); stats[1] = ix->coalescer.requests.load(); }
    return B200VS_OK;
  });
}

int b200vs_range_search(b200vs_index* h, int64_t nq, const float* xq, float radius, int32_t max_results,
                        const b200vs_search_params* sp, float* out_dist, int64_t* out_ids, int32_t* out_counts) {
  return range_search(h, nq, xq, radius, max_results, sp, out_dist, out_ids, out_counts, false);
}

int b200vs_reconstruct(b200vs_index* h, int64_t n, const int64_t* ids, float* out, uint8_t* found) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    if (n <= 0) return B200VS_OK;
    if (!ids || !out) fail(B200VS_EILLEGAL_PARAMETERS, "null ids / output");
    ix->reconstruct(n, ids, out, found);
    return B200VS_OK;
  });
}
int b200vs_sub_type(b200vs_index* h) {
  int r = -1;
  guarded([&]() -> int { IndexBase* ix = get(h); std::shared_lock<std::shared_mutex> rl(ix->rw); r = ix->sub_type(); return B200VS_OK; });
  return r;
}

int b200vs_count(b200vs_index* h, int64_t* count) {
  return guarded([&]() -> int { IndexBase* ix = get(h); std::shared_lock<std::shared_mutex> rl(ix->rw); if (count) *count = ix->count(); return B200VS_OK; });
}
int b200vs_deleted_count(b200vs_index* h, int64_t* count) {
  return guarded([&]() -> int { IndexBase* ix = get(h); std::shared_lock<std::shared_mutex> rl(ix->rw); if (count) *count = ix->deleted_count(); return B200VS_OK; });
}
int b200vs_memory_size(b200vs_index* h, int64_t* bytes) {
  return guarded([&]() -> int { IndexBase* ix = get(h); std::shared_lock<std::shared_mutex> rl(ix->rw); if (bytes) *bytes = ix->memory_size(); return B200VS_OK; });
}
int b200vs_is_trained(b200vs_index* h) {
  int r = 0;
  guarded([&]() -> int { IndexBase* ix = get(h); std::shared_lock<std::shared_mutex> rl(ix->rw); r = ix->is_trained() ? 1 : 0; return B200VS_OK; });
  return r;
}
int32_t b200vs_dimension(b200vs_index* h) { return h && h->impl ? h->impl->dim : -1; }

int b200vs_save(b200vs_index* h, const char* path) {
  return guarded([&]() -> int { if (!path) fail(B200VS_EILLEGAL_PARAMETERS, "null path"); get(h)->save(path); return B200VS_OK; });
}
int b200vs_save_stage(b200vs_index* h) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    h->image.reset();  // a failed stage leaves no image, and the earlier one is not held beside the new one
    SnapshotImage img;
    ix->save_image(img);
    h->image = std::move(img);
    return B200VS_OK;
  });
}
// b200vs_save_staged is in snapshot_write.cc, a host-only translation unit: it runs in a forked child
void b200vs_save_unstage(b200vs_index* h) {
  if (h) h->image.reset();
}
int b200vs_load(b200vs_index* h, const char* path) {
  return guarded([&]() -> int {
    if (!path) fail(B200VS_EILLEGAL_PARAMETERS, "null path");
    IndexBase* ix = get(h);
    ix->load(path);
    std::unique_lock<std::shared_mutex> wl(ix->rw);
    ix->train_rows = ix->count();  // train_data_size_ = ntotal, vector_index_ivf_flat.cc:503-504
    return B200VS_OK;
  });
}

int b200vs_need_rebuild(b200vs_index* h) {
  int r = 0;
  const int rc = guarded([&]() -> int {
    IndexBase* ix = get(h);
    std::shared_lock<std::shared_mutex> rl(ix->rw);
    r = ix->need_rebuild() ? 1 : 0;
    return B200VS_OK;
  });
  return rc == B200VS_OK ? r : -rc;
}

int b200vs_rebuild_from(b200vs_index* dst_h, b200vs_index* src_h, int64_t* n_rows) {
  return guarded([&]() -> int {
    if (n_rows) *n_rows = 0;
    IndexBase* dst = get(dst_h);
    IndexBase* src = get(src_h);
    if (dst == src) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from: dst and src are the same index");
    // every live row: ids are non-negative, and the bounds are inclusive
    const int64_t n = rebuild_range(dst, {src}, 0, INT64_MAX, false);
    if (n_rows) *n_rows = n;
    return B200VS_OK;
  });
}

int b200vs_rebuild_from_range(b200vs_index* dst_h, int32_t n_src, b200vs_index* const* srcs_h, int64_t id_min, int64_t id_max,
                              int64_t* n_rows) {
  return guarded([&]() -> int {
    if (n_rows) *n_rows = 0;
    if (n_src < 1 || n_src > kRebuildMaxSources || !srcs_h)
      fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from_range: 1 to 16 sources, in a non-null list");
    IndexBase* dst = get(dst_h);
    std::vector<IndexBase*> srcs;
    for (int32_t i = 0; i < n_src; ++i) {
      IndexBase* src = get(srcs_h[i]);
      if (src == dst) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from_range: dst is among the sources");
      if (std::find(srcs.begin(), srcs.end(), src) != srcs.end()) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from_range: a source is listed twice");
      srcs.push_back(src);
    }
    if (id_min > id_max) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from_range: id_min > id_max");
    // [id_min, id_max) as inclusive bounds; id_max - 1 cannot overflow once the range holds an id
    const bool none = id_min == id_max;
    const int64_t n = rebuild_range(dst, srcs, none ? 1 : id_min, none ? 0 : id_max - 1, true);
    if (n_rows) *n_rows = n;
    return B200VS_OK;
  });
}

int b200vs_export_lists(b200vs_index* h, int64_t* list_off, float* vectors, uint8_t* codes, int64_t* ids) {
  return guarded([&]() -> int { get(h)->export_lists(list_off, vectors, codes, ids); return B200VS_OK; });
}

int b200vs_export_list(b200vs_index* h, int32_t list, int64_t cap, float* vectors, int64_t* ids, int64_t* count) {
  return guarded([&]() -> int {
    if (cap < 0) fail(B200VS_EILLEGAL_PARAMETERS, "bad capacity");
    const int64_t n = get(h)->export_list(list, cap, vectors, ids);
    if (count) *count = n;
    return B200VS_OK;
  });
}

int b200vs_merge_topk_device(int32_t device, int32_t nparts, int64_t nq, int32_t k, const float* parts_dist,
                             const int64_t* parts_ids, float* out_dist, int64_t* out_ids, void* stream) {
  return guarded([&]() -> int {
    if (nparts <= 0 || nq <= 0 || k <= 0 || !parts_dist || !parts_ids || !out_dist || !out_ids) fail(B200VS_EILLEGAL_PARAMETERS, "bad merge arguments");
    B200VS_CUDA(cudaSetDevice(device));
    launch_merge_api(nparts, nq, k, parts_dist, (const long long*)parts_ids, out_dist, (long long*)out_ids, (cudaStream_t)stream);
    return B200VS_OK;
  });
}

// ---- VectorCalcDistance: pairwise distance matrix (src/vector/vector_index_utils.cc:48-124, :193-419) ----
int b200vs_calc_distance(int32_t device, int32_t algorithm, b200vs_metric metric, int32_t dim, int64_t nl, const float* left,
                         int64_t nr, const float* right, float* out, float* left_out, float* right_out) {
  return guarded([&]() -> int {
    if (algorithm != B200VS_ALGORITHM_FAISS && algorithm != B200VS_ALGORITHM_HNSWLIB)
      fail(B200VS_EILLEGAL_PARAMETERS, "invalid algorithm type : ALGORITHM_NONE");      // utils.cc:70-76
    if (metric != B200VS_L2 && metric != B200VS_IP && metric != B200VS_COSINE)
      fail(B200VS_EILLEGAL_PARAMETERS, "invalid metric_type type : METRIC_TYPE_NONE");   // utils.cc:151-157
    if (dim <= 0 || nl < 0 || nr < 0) fail(B200VS_EILLEGAL_PARAMETERS, "bad distance-matrix shape");
    if (nl == 0 || nr == 0) return B200VS_OK;  // CalcDistanceCore over empty operands: empty result
    if (!left || !right || !out) fail(B200VS_EILLEGAL_PARAMETERS, "null operand");
    B200VS_CUDA(cudaSetDevice(device));
    cudaStream_t s = nullptr;
    B200VS_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    DevBuf<float> dl, dr, dn, dout;
    try {
      dl.reserve((size_t)nl * dim, 0, s); dr.reserve((size_t)nr * dim, 0, s); dout.reserve((size_t)nl * nr, 0, s);
      B200VS_CUDA(cudaMemcpyAsync(dl.p, left, (size_t)nl * dim * 4, cudaMemcpyHostToDevice, s));
      B200VS_CUDA(cudaMemcpyAsync(dr.p, right, (size_t)nr * dim * 4, cudaMemcpyHostToDevice, s));
      if (metric == B200VS_COSINE) {
        if (algorithm == B200VS_ALGORITHM_FAISS) {  // NormalizeVectorForFaiss on copies, utils.cc:283-284
          launch_normalize_faiss(dl.p, nl, dim, s);
          launch_normalize_faiss(dr.p, nr, dim, s);
        } else {                                    // NormalizeVectorForHnsw, utils.cc:407-413 (out of place)
          dn.reserve((size_t)std::max(nl, nr) * dim, 0, s);
          launch_normalize_hnsw(dl.p, dn.p, nl, dim, s);
          B200VS_CUDA(cudaMemcpyAsync(dl.p, dn.p, (size_t)nl * dim * 4, cudaMemcpyDeviceToDevice, s));
          launch_normalize_hnsw(dr.p, dn.p, nr, dim, s);
          B200VS_CUDA(cudaMemcpyAsync(dr.p, dn.p, (size_t)nr * dim * 4, cudaMemcpyDeviceToDevice, s));
        }
      }
      launch_pair_distance(metric == B200VS_L2, dl.p, nl, dr.p, nr, dim, dout.p, s);
      B200VS_CUDA(cudaMemcpyAsync(out, dout.p, (size_t)nl * nr * 4, cudaMemcpyDeviceToHost, s));
      if (left_out) B200VS_CUDA(cudaMemcpyAsync(left_out, dl.p, (size_t)nl * dim * 4, cudaMemcpyDeviceToHost, s));
      if (right_out) B200VS_CUDA(cudaMemcpyAsync(right_out, dr.p, (size_t)nr * dim * 4, cudaMemcpyDeviceToHost, s));
      B200VS_CUDA(cudaStreamSynchronize(s));
    } catch (...) {
      cudaStreamSynchronize(s); dl.free(); dr.free(); dn.free(); dout.free(); cudaStreamDestroy(s);
      throw;
    }
    dl.free(); dr.free(); dn.free(); dout.free();
    cudaStreamDestroy(s);
    return B200VS_OK;
  });
}

// CalcHammingDistanceByFaiss (vector_index_utils.cc:333-357): packed rows zero-padded to 32-bit words, then the pair kernel
// with the Hamming functor
int b200vs_calc_distance_binary(int32_t device, int32_t nbytes, int64_t nl, const uint8_t* left, int64_t nr, const uint8_t* right,
                                float* out) {
  return guarded([&]() -> int {
    if (nbytes <= 0 || nbytes > 4096) fail(B200VS_EILLEGAL_PARAMETERS, "binary row size must be in (0, 4096] bytes");
    if (nl < 0 || nr < 0) fail(B200VS_EILLEGAL_PARAMETERS, "bad distance-matrix shape");
    if (nl == 0 || nr == 0) return B200VS_OK;
    if (!left || !right || !out) fail(B200VS_EILLEGAL_PARAMETERS, "null operand");
    const int w = (nbytes + 3) / 4;
    B200VS_CUDA(cudaSetDevice(device));
    cudaStream_t s = nullptr;
    B200VS_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    DevBuf<uint8_t> raw;
    DevBuf<uint32_t> wl, wr;
    DevBuf<float> dout;
    try {
      raw.reserve((size_t)std::max(nl, nr) * nbytes, 0, s);
      wl.reserve((size_t)nl * w, 0, s); wr.reserve((size_t)nr * w, 0, s); dout.reserve((size_t)nl * nr, 0, s);
      B200VS_CUDA(cudaMemcpyAsync(raw.p, left, (size_t)nl * nbytes, cudaMemcpyHostToDevice, s));
      launch_pad_rows(raw.p, nl, nbytes, wl.p, s);
      B200VS_CUDA(cudaMemcpyAsync(raw.p, right, (size_t)nr * nbytes, cudaMemcpyHostToDevice, s));
      launch_pad_rows(raw.p, nr, nbytes, wr.p, s);
      launch_pair_hamming(wl.p, nl, wr.p, nr, w, dout.p, s);
      B200VS_CUDA(cudaMemcpyAsync(out, dout.p, (size_t)nl * nr * 4, cudaMemcpyDeviceToHost, s));
      B200VS_CUDA(cudaStreamSynchronize(s));
    } catch (...) {
      cudaStreamSynchronize(s); raw.free(); wl.free(); wr.free(); dout.free(); cudaStreamDestroy(s);
      throw;
    }
    raw.free(); wl.free(); wr.free(); dout.free();
    cudaStreamDestroy(s);
    return B200VS_OK;
  });
}

// ---- streaming brute-force scan: VectorReader::BruteForceSearch (src/vector/vector_reader.cc:1873-2048) ----
struct b200vs_scan {
  IndexBase* flat = nullptr;  // one tile at a time
  int64_t nq = 0;
  int k = 0;
  bool has_sp = false;
  b200vs_search_params sp{};
  std::vector<int64_t> allow;  // private copy of sp.sorted_ids (the caller's array need not outlive scan_begin)
  cudaStream_t s = nullptr;
  DevBuf<float> q, parts_d, out_d;      // parts = [2, nq, k]: running result, tile result
  DevBuf<long long> parts_i, out_i;
  bool deep = false;                    // k past the exact scan's shared-memory select: tiles and merge on the deep path
  DevBuf<float> cat_d;                  // deep merge input [nq, 2k]: each query's running result, then its tile result
  DevBuf<long long> cat_i;
  int64_t pushed = 0;
  ~b200vs_scan() {
    if (flat) { cudaSetDevice(flat->device); }
    if (s) cudaStreamSynchronize(s);
    q.free(); parts_d.free(); out_d.free(); parts_i.free(); out_i.free(); cat_d.free(); cat_i.free();
    delete flat;
    if (s) cudaStreamDestroy(s);
  }
};

int b200vs_scan_begin(int32_t device, b200vs_metric metric, int32_t dim, int64_t nq, const float* xq, int32_t k,
                      const b200vs_search_params* sp, b200vs_scan** out) {
  return guarded([&]() -> int {
    if (!out) fail(B200VS_EILLEGAL_PARAMETERS, "out is null");
    *out = nullptr;
    if (dim <= 0) fail(B200VS_EVECTOR_INVALID, "vector index dimension is invalid");  // vector_reader.cc:1889-1894
    if (metric == B200VS_HAMMING) fail(B200VS_EVECTOR_NOT_SUPPORT, "brute-force scan of binary vectors is not implemented");
    if (metric != B200VS_L2 && metric != B200VS_IP && metric != B200VS_COSINE) fail(B200VS_EILLEGAL_PARAMETERS, "unsupported metric type");
    if (nq <= 0 || !xq) fail(B200VS_EILLEGAL_PARAMETERS, "vector_with_ids is empty");
    if (k <= 0) fail(B200VS_EILLEGAL_PARAMETERS, "topk must be > 0");
    b200vs_params p{};
    p.device = device;
    std::unique_ptr<b200vs_scan> st(new b200vs_scan());
    st->flat = make_flat(metric, dim, p);
    st->nq = nq; st->k = k;
    st->deep = !exact_select_fits(dim, 1, k);
    if (st->deep && k > kDeepMaxK) fail(B200VS_EILLEGAL_PARAMETERS, "topk above " + std::to_string(kDeepMaxK));
    if (sp) {
      st->has_sp = true; st->sp = *sp;
      if (sp->sorted_ids && sp->n_ids > 0) st->allow.assign(sp->sorted_ids, sp->sorted_ids + sp->n_ids);
      st->sp.sorted_ids = sp->sorted_ids ? st->allow.data() : nullptr;
    }
    B200VS_CUDA(cudaSetDevice(device));
    B200VS_CUDA(cudaStreamCreateWithFlags(&st->s, cudaStreamNonBlocking));
    const size_t nk = (size_t)nq * k;
    st->q.reserve((size_t)nq * dim, 0, st->s);
    st->parts_d.reserve(2 * nk, 0, st->s); st->parts_i.reserve(2 * nk, 0, st->s);
    st->out_d.reserve(nk, 0, st->s); st->out_i.reserve(nk, 0, st->s);
    if (st->deep) { st->cat_d.reserve(2 * nk, 0, st->s); st->cat_i.reserve(2 * nk, 0, st->s); }
    B200VS_CUDA(cudaMemcpyAsync(st->q.p, xq, (size_t)nq * dim * 4, cudaMemcpyHostToDevice, st->s));
    B200VS_CUDA(cudaMemsetAsync(st->parts_d.p, 0, 2 * nk * 4, st->s));
    B200VS_CUDA(cudaMemsetAsync(st->parts_i.p, 0xFF, 2 * nk * 8, st->s));  // id -1 = empty slot
    B200VS_CUDA(cudaStreamSynchronize(st->s));
    *out = st.release();
    return B200VS_OK;
  });
}

int b200vs_scan_push(b200vs_scan* st, int64_t n, const float* x, const int64_t* ids) {
  return guarded([&]() -> int {
    if (!st || !st->flat) fail(B200VS_EILLEGAL_PARAMETERS, "null scan handle");
    if (n <= 0) return B200VS_OK;
    if (!x || !ids) fail(B200VS_EILLEGAL_PARAMETERS, "null tile");
    IndexBase* ix = st->flat;
    const size_t nk = (size_t)st->nq * st->k;
    check_ids_nonnegative(n, ids);  // before the previous tile is cleared
    if (st->pushed > 0) ix->clear();
    ix->add(AddReq::host(n, x, ids));  // one temporary Flat index per tile, as the reference builds (vector_reader.cc:1937-1946)
    index_read(ix, st->s, st->has_sp ? &st->sp : nullptr, [&](const SearchCtx& sc, cudaStream_t s) {
      SearchReq r;
      r.nq = st->nq; r.xq = st->q.p; r.k = st->k; r.sc = &sc; r.od = st->parts_d.p + nk; r.oi = st->parts_i.p + nk; r.deep = st->deep;
      ix->search(r, s);
      if (!st->deep) return;
      // running top-k <- the deep select over each query's 2k slots [running, tile]
      const size_t k = (size_t)st->k;
      for (int part = 0; part < 2; ++part) {
        B200VS_CUDA(cudaMemcpy2DAsync(st->cat_d.p + part * k, 2 * k * 4, st->parts_d.p + part * nk, k * 4, k * 4, (size_t)st->nq,
                                      cudaMemcpyDeviceToDevice, s));
        B200VS_CUDA(cudaMemcpy2DAsync(st->cat_i.p + part * k, 2 * k * 8, st->parts_i.p + part * nk, k * 8, k * 8, (size_t)st->nq,
                                      cudaMemcpyDeviceToDevice, s));
      }
      run_deep_merge_api(ix, st->nq, st->k, 2 * st->k, st->cat_d.p, st->cat_i.p, st->out_d.p, st->out_i.p, s);
    });
    // running top-k <- merge(running, tile): the reference's per-query priority queues (:1956-1971)
    if (!st->deep) launch_merge_api(2, st->nq, st->k, st->parts_d.p, st->parts_i.p, st->out_d.p, st->out_i.p, st->s);
    B200VS_CUDA(cudaMemcpyAsync(st->parts_d.p, st->out_d.p, nk * 4, cudaMemcpyDeviceToDevice, st->s));
    B200VS_CUDA(cudaMemcpyAsync(st->parts_i.p, st->out_i.p, nk * 8, cudaMemcpyDeviceToDevice, st->s));
    B200VS_CUDA(cudaStreamSynchronize(st->s));  // the next push rewrites the tile index
    st->pushed += n;
    return B200VS_OK;
  });
}

int b200vs_scan_finish(b200vs_scan* st, float* out_dist, int64_t* out_ids) {
  const int rc = guarded([&]() -> int {
    if (!st || !st->flat) fail(B200VS_EILLEGAL_PARAMETERS, "null scan handle");
    if (!out_dist || !out_ids) fail(B200VS_EILLEGAL_PARAMETERS, "null output");
    B200VS_CUDA(cudaSetDevice(st->flat->device));
    const size_t nk = (size_t)st->nq * st->k;
    B200VS_CUDA(cudaMemcpyAsync(out_dist, st->parts_d.p, nk * 4, cudaMemcpyDeviceToHost, st->s));
    B200VS_CUDA(cudaMemcpyAsync(out_ids, st->parts_i.p, nk * 8, cudaMemcpyDeviceToHost, st->s));
    B200VS_CUDA(cudaStreamSynchronize(st->s));
    return B200VS_OK;
  });
  delete st;
  return rc;
}

void b200vs_scan_abort(b200vs_scan* st) { delete st; }

// ---- streaming brute-force range scan: VectorReader::BruteForceRangeSearch (src/vector/vector_reader.cc:2050-2202) ----
// No temporary index: each pushed tile goes straight to range_append_kernel, which appends its hits in row order.
struct b200vs_scan_range {
  int device = 0;
  int dim = 0;
  int64_t nq = 0;
  int max_results = 0;
  bool l2 = true, cosine = false;
  bool no_hits = false;  // a NaN radius: no row is a hit, so pushes launch nothing
  float thr_raw = 0;  // L2: dist < radius; IP / cosine: ip > 1 - radius (vector_index_flat.cc:282-285)
  SearchCtx sc;       // sc.sorted_ids_dev points into allow
  cudaStream_t s = nullptr;
  DevBuf<float> q, x, out_d;  // queries [nq, dim], tile [rows, dim], results [nq, max_results]
  DevBuf<long long> ids, allow, out_i;
  DevBuf<int> counts;         // [nq] hits kept so far
  ~b200vs_scan_range() {
    cudaSetDevice(device);
    if (s) cudaStreamSynchronize(s);
    q.free(); x.free(); out_d.free(); ids.free(); allow.free(); out_i.free(); counts.free();
    if (s) cudaStreamDestroy(s);
  }
};

int b200vs_scan_range_begin(int32_t device, b200vs_metric metric, int32_t dim, int64_t nq, const float* xq, float radius,
                            int32_t max_results, const b200vs_search_params* sp, b200vs_scan_range** out) {
  return guarded([&]() -> int {
    if (!out) fail(B200VS_EILLEGAL_PARAMETERS, "out is null");
    *out = nullptr;
    if (dim <= 0) fail(B200VS_EVECTOR_INVALID, "vector index dimension is invalid");  // as b200vs_scan_begin
    if (metric == B200VS_HAMMING) fail(B200VS_EVECTOR_NOT_SUPPORT, "brute-force scan of binary vectors is not implemented");
    if (metric != B200VS_L2 && metric != B200VS_IP && metric != B200VS_COSINE) fail(B200VS_EILLEGAL_PARAMETERS, "unsupported metric type");
    if (nq <= 0 || !xq) fail(B200VS_EILLEGAL_PARAMETERS, "vector_with_ids is empty");
    if (max_results <= 0) fail(B200VS_EILLEGAL_PARAMETERS, "max_results must be > 0");
    std::unique_ptr<b200vs_scan_range> st(new b200vs_scan_range());
    st->device = device; st->dim = dim; st->nq = nq; st->max_results = max_results;
    st->l2 = metric == B200VS_L2;
    st->cosine = metric == B200VS_COSINE;
    st->thr_raw = st->l2 ? radius : 1.0F - radius;
    st->no_hits = std::isnan(radius);
    B200VS_CUDA(cudaSetDevice(device));
    B200VS_CUDA(cudaStreamCreateWithFlags(&st->s, cudaStreamNonBlocking));
    const size_t nr = (size_t)nq * max_results;
    st->q.reserve((size_t)nq * dim, 0, st->s);
    st->out_d.reserve(nr, 0, st->s); st->out_i.reserve(nr, 0, st->s); st->counts.reserve((size_t)nq, 0, st->s);
    if (sp) {  // the filters as make_ctx resolves them for an index search, copied: the caller's list need not outlive begin
      st->sc.has_range = sp->has_range; st->sc.negate = sp->negate; st->sc.rmin = sp->range_min; st->sc.rmax = sp->range_max;
      if (sp->sorted_ids) {
        st->allow.reserve((size_t)std::max<int64_t>(sp->n_ids, 1), 0, st->s);
        if (sp->n_ids > 0) B200VS_CUDA(cudaMemcpyAsync(st->allow.p, sp->sorted_ids, (size_t)sp->n_ids * 8, cudaMemcpyHostToDevice, st->s));
        st->sc.sorted_ids_dev = st->allow.p;
        st->sc.n_ids = sp->n_ids;
      }
    }
    B200VS_CUDA(cudaMemcpyAsync(st->q.p, xq, (size_t)nq * dim * 4, cudaMemcpyHostToDevice, st->s));
    if (st->cosine) launch_normalize_faiss(st->q.p, nq, dim, st->s);  // NormalizeVectorForFaiss, as a Flat index searches
    B200VS_CUDA(cudaMemsetAsync(st->out_d.p, 0, nr * 4, st->s));
    B200VS_CUDA(cudaMemsetAsync(st->out_i.p, 0xFF, nr * 8, st->s));  // id -1 = empty slot
    B200VS_CUDA(cudaMemsetAsync(st->counts.p, 0, (size_t)nq * 4, st->s));
    B200VS_CUDA(cudaStreamSynchronize(st->s));
    *out = st.release();
    return B200VS_OK;
  });
}

int b200vs_scan_range_push(b200vs_scan_range* st, int64_t n, const float* x, const int64_t* ids) {
  return guarded([&]() -> int {
    if (!st) fail(B200VS_EILLEGAL_PARAMETERS, "null scan handle");
    if (n <= 0) return B200VS_OK;
    if (!x || !ids) fail(B200VS_EILLEGAL_PARAMETERS, "null tile");
    check_batch_ids_unique(n, ids);  // the Flat add of the reference's per-tile index refuses a repeated id
    if (st->no_hits) return B200VS_OK;
    B200VS_CUDA(cudaSetDevice(st->device));
    st->x.reserve((size_t)n * st->dim, 0, st->s);
    st->ids.reserve((size_t)n, 0, st->s);
    B200VS_CUDA(cudaMemcpyAsync(st->x.p, x, (size_t)n * st->dim * 4, cudaMemcpyHostToDevice, st->s));
    B200VS_CUDA(cudaMemcpyAsync(st->ids.p, ids, (size_t)n * 8, cudaMemcpyHostToDevice, st->s));
    if (st->cosine) launch_normalize_faiss(st->x.p, n, st->dim, st->s);  // vector_index_flat.cc:155
    launch_range_append(st->l2, st->x.p, st->ids.p, nullptr, n, st->dim, st->nq, st->q.p, st->sc, st->thr_raw, st->max_results,
                        st->out_d.p, st->out_i.p, st->counts.p, st->s);
    B200VS_CUDA(cudaStreamSynchronize(st->s));  // the caller may reuse its buffers, and the next push rewrites the tile
    return B200VS_OK;
  });
}

int b200vs_scan_range_finish(b200vs_scan_range* st, float* out_dist, int64_t* out_ids, int32_t* out_counts) {
  const int rc = guarded([&]() -> int {
    if (!st) fail(B200VS_EILLEGAL_PARAMETERS, "null scan handle");
    if (!out_dist || !out_ids || !out_counts) fail(B200VS_EILLEGAL_PARAMETERS, "null output");
    B200VS_CUDA(cudaSetDevice(st->device));
    const size_t nr = (size_t)st->nq * st->max_results;
    B200VS_CUDA(cudaMemcpyAsync(out_dist, st->out_d.p, nr * 4, cudaMemcpyDeviceToHost, st->s));
    B200VS_CUDA(cudaMemcpyAsync(out_ids, st->out_i.p, nr * 8, cudaMemcpyDeviceToHost, st->s));
    B200VS_CUDA(cudaMemcpyAsync(out_counts, st->counts.p, (size_t)st->nq * 4, cudaMemcpyDeviceToHost, st->s));
    B200VS_CUDA(cudaStreamSynchronize(st->s));
    return B200VS_OK;
  });
  delete st;
  return rc;
}

void b200vs_scan_range_abort(b200vs_scan_range* st) { delete st; }

// ---- binary indexes (binary.cu): packed rows, dim / 8 bytes each ----
int b200vs_train_binary(b200vs_index* h, int64_t n, const uint8_t* x) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    check_row_type(ix, true);
    if (n <= 0 || !x) fail(B200VS_EILLEGAL_PARAMETERS, "data size invalid");
    ix->train(n, x);
    return B200VS_OK;
  });
}

int b200vs_add_with_ids_binary(b200vs_index* h, int64_t n, const uint8_t* x, const int64_t* ids, int upsert) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    check_row_type(ix, true);
    if (n <= 0 || !x || !ids) fail(B200VS_EILLEGAL_PARAMETERS, "vector_with_ids is empty");
    ix->add(AddReq::host(n, x, ids, upsert != 0));
    return B200VS_OK;
  });
}

int b200vs_search_binary_device(b200vs_index* h, int64_t nq, const uint8_t* xq_dev, int32_t k, const b200vs_search_params* sp,
                                float* out_dist_dev, int64_t* out_ids_dev, void* stream) {
  return search_device(h, nq, xq_dev, k, sp, out_dist_dev, out_ids_dev, stream, true);
}

int b200vs_search_binary(b200vs_index* h, int64_t nq, const uint8_t* xq, int32_t k, const b200vs_search_params* sp, float* out_dist,
                         int64_t* out_ids) {
  return host_search(h, nq, xq, k, sp, out_dist, out_ids, true);
}

int b200vs_range_search_binary(b200vs_index* h, int64_t nq, const uint8_t* xq, float radius, int32_t max_results,
                               const b200vs_search_params* sp, float* out_dist, int64_t* out_ids, int32_t* out_counts) {
  return range_search(h, nq, xq, radius, max_results, sp, out_dist, out_ids, out_counts, true);
}

int b200vs_last_phase_times(b200vs_index* h, float ms[16]) {
  return guarded([&]() -> int {
    IndexBase* ix = get(h);
    for (int i = 0; i < 16; ++i) ms[i] = i < IndexBase::PH_COUNT ? ix->phase_ms[i] : 0.f;
    return B200VS_OK;
  });
}

int b200vs_last_search_stats(b200vs_index* h, int64_t stats[8]) {
  return guarded([&]() -> int { IndexBase* ix = get(h); for (int i = 0; i < 8; ++i) stats[i] = ix->stats[i]; return B200VS_OK; });
}

int b200vs_set_profiling(b200vs_index* h, int on) {
  return guarded([&]() -> int { get(h)->profiling = on != 0; return B200VS_OK; });
}

const char* b200vs_last_error(void) { return g_last_error.c_str(); }
const char* b200vs_version(void) { return "b200vs 0.1 (sm_90a)"; }

}  // extern "C"
