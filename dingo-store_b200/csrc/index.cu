// index.cu — IndexBase, FlatIndex, IvfFlatIndex (device-resident replacements of the faiss objects held by
// VectorIndexFlat / VectorIndexIvfFlat, src/vector/vector_index_flat.cc:73-107, vector_index_ivf_flat.cc:805-837).
#include <algorithm>
#include <cstdio>
#include <random>
#include <unordered_set>

#include "index.h"
#include "ivf_common.h"
#include "flat_small.cuh"
#include "tc_scan.cuh"

namespace b200vs {

thread_local std::string g_last_error;
thread_local Lane* IndexBase::tl_lane = nullptr;
thread_local IndexBase* IndexBase::tl_owner = nullptr;
thread_local const IndexBase* RwSharedGuard::tl_held = nullptr;

LaneGuard::LaneGuard(IndexBase* ix_, cudaStream_t s) : ix(ix_), lane(nullptr), prev_owner(IndexBase::tl_owner), prev_lane(IndexBase::tl_lane), stream(s) {
  const bool own = s == nullptr;  // host-pointer / NULL-stream call: runs on the lane's own stream
  {
    std::lock_guard<std::mutex> pick(ix->lane_pick_mu);
    // 1) the lane this stream used last: its scratch is already ordered behind the caller's earlier work
    if (!own)
      for (auto& l : ix->lanes)
        if (l.last.load() == s && l.mu.try_lock()) { lane = &l; break; }
    // 2) a free lane nobody else's stream is attached to: for host-pointer calls the most recently used such lane
    //    (its scratch arena is already sized and hot), else an unused one; failing that, steal the least recently used
    if (!lane) {
      auto rank = [&](Lane& l) -> unsigned long long {
        const cudaStream_t last = l.last.load();
        if (own && last != nullptr && last == l.own) return (1ull << 60) - l.tick;  // warm host-call lane, MRU first
        if (last == nullptr) return 1ull << 61;                                       // never used
        return (1ull << 62) + l.tick;                                                 // attached to a stream: LRU
      };
      for (auto& l : ix->lanes) {
        if (!l.mu.try_lock()) continue;
        if (!lane) lane = &l;
        else if (rank(l) < rank(*lane)) { lane->mu.unlock(); lane = &l; }
        else l.mu.unlock();
      }
    }
    if (lane) lane->tick = ++ix->lane_tick;
  }
  if (!lane) {  // every lane is busy: queue behind one
    lane = &ix->lanes[ix->lane_rr.fetch_add(1) % kLanes];
    lane->mu.lock();
    std::lock_guard<std::mutex> pick(ix->lane_pick_mu);
    lane->tick = ++ix->lane_tick;
  }
  try {
    if (own) {
      if (!lane->own) B200VS_CUDA(cudaStreamCreateWithFlags(&lane->own, cudaStreamNonBlocking));
      stream = lane->own;
    }
    if (lane->last.load() != stream && lane->done_valid.load()) B200VS_CUDA(cudaStreamWaitEvent(stream, lane->done, 0));
    lane->last.store(stream);
    IndexBase::tl_owner = ix;
    IndexBase::tl_lane = lane;
    if (lane->s.buf.cap == 0) {  // first search on this lane: size its arena like the largest warmed-up lane, so it does
      size_t want = 0;            // not go through overflow blocks + consolidation (cudaFree = device-wide stalls)
      for (auto& l : ix->lanes) want = std::max(want, l.s.buf.cap);
      if (want) lane->s.buf.reserve(want, 0, stream);
    }
    lane->s.reset(stream);
  } catch (...) {
    IndexBase::tl_owner = prev_owner;
    IndexBase::tl_lane = prev_lane;
    lane->mu.unlock();
    throw;
  }
}
LaneGuard::~LaneGuard() {
  IndexBase::tl_owner = prev_owner;
  IndexBase::tl_lane = prev_lane;
  if (!lane->done) cudaEventCreateWithFlags(&lane->done, cudaEventDisableTiming);
  if (lane->done && cudaEventRecord(lane->done, stream) == cudaSuccess) lane->done_valid.store(true);
  lane->mu.unlock();
}

IndexBase::IndexBase(b200vs_type t, b200vs_metric m, int d, const b200vs_params& p)
    : type(t), metric(m), dim(d), device(p.device), params(p) {
  set_device();
  B200VS_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  last_stream = stream;
}
IndexBase::~IndexBase() {
  cudaSetDevice(device);
  if (stream) { cudaStreamSynchronize(stream); cudaStreamDestroy(stream); }
  for (auto& l : lanes) {
    if (l.done) { cudaEventSynchronize(l.done); cudaEventDestroy(l.done); }
    if (l.own) { cudaStreamSynchronize(l.own); cudaStreamDestroy(l.own); }
  }
}

SearchCtx make_ctx(IndexBase* ix, const b200vs_search_params* sp, cudaStream_t s) {
  SearchCtx sc;
  if (!sp) return sc;
  sc.nprobe = sp->nprobe;
  sc.efsearch = sp->efsearch;
  sc.exact_only = sp->exact_only;
  sc.has_range = sp->has_range;
  sc.negate = sp->negate;
  sc.rmin = sp->range_min;
  sc.rmax = sp->range_max;
  if (sp->sorted_ids) {
    long long* d = ix->scratch.alloc<long long>((size_t)std::max<int64_t>(sp->n_ids, 1));
    if (sp->n_ids > 0) B200VS_CUDA(cudaMemcpyAsync(d, sp->sorted_ids, (size_t)sp->n_ids * 8, cudaMemcpyHostToDevice, s));
    sc.sorted_ids_dev = d;
    sc.n_ids = sp->n_ids;
  }
  return sc;
}

const float* IndexBase::prepare_queries(int64_t nq, const float* xq_dev, cudaStream_t s) {
  if (metric != B200VS_COSINE) return xq_dev;
  float* q = scratch.alloc<float>((size_t)nq * dim);
  if (type == B200VS_HNSW) {  // NormalizeVectorForHnsw, vector_index_hnsw.cc:449-452
    launch_normalize_hnsw(xq_dev, q, nq, dim, s);
  } else {                    // NormalizeVectorForFaiss via ExtractVectorValue(normalize_), flat.cc:243
    B200VS_CUDA(cudaMemcpyAsync(q, xq_dev, (size_t)nq * dim * sizeof(float), cudaMemcpyDeviceToDevice, s));
    launch_normalize_faiss(q, nq, dim, s);
  }
  launch_count(1);
  return q;
}

// Save / Load (VectorIndex::Save/Load, src/vector/vector_index.h:168-170; reference: faiss::write_index / read_index at
// vector_index_flat.cc:354,:379, write_index_binary, and hnswlib saveIndex at vector_index_hnsw.cc:290).  Own container, not
// faiss-compatible (SURVEY 8f-4): header, trained-state blob, list offsets, ids, then the live rows in list-major order
// exactly as stored.  Float indexes ("B2VSIDX1") store FP32 rows, binary ones ("B2VSBIN1") packed rows of dim / 8 bytes.
namespace {
using FileHdr = IndexFileHdr;
void wr(FILE* f, const void* p, size_t n) { if (n && fwrite(p, 1, n, f) != n) fail(B200VS_EINTERNAL, "short write"); }
void rd(FILE* f, void* p, size_t n) { if (n && fread(p, 1, n, f) != n) fail(B200VS_EINTERNAL, "short read / truncated index file"); }
}  // namespace

void IndexBase::save(const std::string& path) {
  RwSharedGuard hold(this);  // one reader hold across count / trained state / export: no add can slip in between
  const int64_t st_len = get_state(nullptr, 0);
  std::vector<unsigned char> st((size_t)std::max<int64_t>(st_len, 0));
  if (st_len > 0) get_state(st.data(), st.size());
  const int nl = export_nlist();
  const int64_t n = type == B200VS_HNSW ? 0 : count();  // the HNSW blob already carries rows + labels
  const size_t rb = query_row_bytes();
  std::vector<int64_t> off(nl + 1, 0), ids((size_t)n);
  std::vector<uint8_t> rows((size_t)n * rb);
  if (n && binary()) export_lists(off.data(), nullptr, rows.data(), ids.data());
  else if (n) export_lists(off.data(), reinterpret_cast<float*>(rows.data()), nullptr, ids.data());
  FILE* f = fopen(path.c_str(), "wb");
  if (!f) fail(B200VS_EINTERNAL, "cannot open " + path);
  try {
    FileHdr h;
    memcpy(h.magic, binary() ? "B2VSBIN1" : "B2VSIDX1", 8);
    h.type = type; h.metric = metric; h.dim = dim; h.nlist = nl; h.state_len = st_len > 0 ? st_len : 0; h.count = n;
    wr(f, &h, sizeof(h));
    wr(f, st.data(), st.size());
    wr(f, off.data(), off.size() * 8);
    wr(f, ids.data(), ids.size() * 8);
    wr(f, rows.data(), rows.size());
  } catch (...) { fclose(f); throw; }
  fclose(f);
}

void IndexBase::load(const std::string& path) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) fail(B200VS_EINTERNAL, "cannot open " + path);
  try {
    FileHdr h;
    rd(f, &h, sizeof(h));
    if (memcmp(h.magic, binary() ? "B2VSBIN1" : "B2VSIDX1", 8) != 0 || h.type != (int)type || h.metric != (int)metric || h.dim != dim)
      fail(B200VS_EINTERNAL, "index file does not match this index (type / metric / dimension)");
    if (count() != 0) fail(B200VS_EINTERNAL, "load into a non-empty index");
    const size_t rb = query_row_bytes();
    {  // the header's sizes must fit the file before anything is allocated from them
      const long here = ftell(f);
      fseek(f, 0, SEEK_END);
      const long fsize = ftell(f);
      fseek(f, here, SEEK_SET);
      const double need = (double)h.state_len + ((double)h.nlist + 1) * 8 + (double)h.count * (8 + (double)rb);
      if (h.state_len < 0 || h.count < 0 || h.nlist < 0 || h.nlist > (1 << 24) || need > (double)(fsize - here))
        fail(B200VS_EINTERNAL, "corrupt index file (header sizes exceed the file)");
    }
    std::vector<unsigned char> st((size_t)h.state_len);
    rd(f, st.data(), st.size());
    if (h.state_len > 0) set_state(st.data(), st.size());
    std::vector<int64_t> off((size_t)h.nlist + 1), ids((size_t)h.count);
    std::vector<uint8_t> rows((size_t)h.count * rb);
    rd(f, off.data(), off.size() * 8);
    rd(f, ids.data(), ids.size() * 8);
    rd(f, rows.data(), rows.size());
    // the rows come back exactly as stored, each into the list it was saved in (a row added to a caller's list need not
    // be in its nearest list, so the lists are not assigned again)
    std::vector<long long> h_list;
    if (h.nlist > 1) {
      if (off[0] != 0 || off[h.nlist] != h.count || !std::is_sorted(off.begin(), off.end())) fail(B200VS_EINTERNAL, "corrupt index file (list offsets)");
      h_list.resize((size_t)h.count);
      for (int l = 0; l < h.nlist; ++l) std::fill(h_list.begin() + off[l], h_list.begin() + off[l + 1], (long long)l);
    }
    DevBuf<unsigned char> dx;
    DevBuf<long long> dids, dlist;
    for (int64_t a = 0; a < h.count; a += 32768) {
      const int64_t m = std::min<int64_t>(32768, h.count - a);
      if (h_list.empty()) {
        add(AddReq::host(m, rows.data() + (size_t)a * rb, ids.data() + a, false, AddReq::PREPARED));
        continue;
      }
      set_device();
      dx.reserve((size_t)m * rb, 0, stream); dids.reserve(m, 0, stream); dlist.reserve(m, 0, stream);
      B200VS_CUDA(cudaMemcpy(dx.p, rows.data() + (size_t)a * rb, (size_t)m * rb, cudaMemcpyHostToDevice));
      B200VS_CUDA(cudaMemcpy(dids.p, ids.data() + a, (size_t)m * 8, cudaMemcpyHostToDevice));
      B200VS_CUDA(cudaMemcpy(dlist.p, h_list.data() + a, (size_t)m * 8, cudaMemcpyHostToDevice));
      AddReq r = AddReq::device(m, dx.p, dids.p, dlist.p, false, AddReq::PREPARED);
      r.ids = ids.data() + a;
      add(r);
    }
  } catch (...) { fclose(f); throw; }
  fclose(f);
}

void IndexBase::stage(const AddReq& r, size_t row_bytes, bool own, Staged& st) {
  st.x = const_cast<void*>(r.x);
  st.ids_dev = r.ids_dev;
  st.ids = r.ids;
  if (!r.on_device || own) {
    st.x = scratch.alloc<unsigned char>((size_t)r.n * row_bytes);
    B200VS_CUDA(cudaMemcpyAsync(st.x, r.x, (size_t)r.n * row_bytes, r.on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, stream));
  }
  if (!r.on_device) {
    long long* d = scratch.alloc<long long>(r.n);
    B200VS_CUDA(cudaMemcpyAsync(d, r.ids, (size_t)r.n * 8, cudaMemcpyHostToDevice, stream));
    st.ids_dev = d;
  } else if (!r.ids) {
    st.ids_buf.resize(r.n);
    B200VS_CUDA(cudaMemcpyAsync(st.ids_buf.data(), r.ids_dev, (size_t)r.n * 8, cudaMemcpyDeviceToHost, stream));
    B200VS_CUDA(cudaStreamSynchronize(stream));
    st.ids = st.ids_buf.data();
  }
  check_ids_nonnegative(r.n, st.ids);
}

void check_batch_ids_unique(int64_t n, const int64_t* ids) {  // CheckVectorIdDuplicated, vector_index_utils.cc:551-561
  std::unordered_set<int64_t> seen;
  seen.reserve((size_t)n * 2);
  for (int64_t i = 0; i < n; ++i)
    if (!seen.insert(ids[i]).second) fail(B200VS_EVECTOR_ID_DUPLICATED, "vector id duplicated: " + std::to_string(ids[i]));
}

// ============================================================================================
// Device rows of a Flat index or an IVF-Flat arena: FP32 rows, ids (-1 = tombstone / unused slot), ||x||^2 and, when
// the owner asks for it and dim % 8 == 0 (16-byte FP16 row pitch for TMA), the FP16 mirror the tile list scan streams
// instead of the FP32 rows (DESIGN.md 3, 4.2).  Every write of the rows goes through here, so the arrays stay in step.
// The owner decides capacities and slots; the store moves rows.  All work runs on the owner's stream.
// ============================================================================================
struct RowStore {
  IndexBase* const ix;     // scratch for the device copies of host-side row lists
  const int d;
  const cudaStream_t s;
  const bool want_mirror;
  DevBuf<float> vecs;      // [cap, d]
  DevBuf<long long> ids;   // [cap]
  DevBuf<float> norms;     // [cap]
  DevBuf<__half> vecs_h;   // [cap, d]  RN(x * 2^-e) per row
  DevBuf<float> hscale;    // [cap]     2^e
  bool mirror;             // the mirror is kept: wanted, and no allocation of it failed since the last reset()
  float max_norm = 0.f;    // max ||x|| over every row written: grows only (tc_eps)

  RowStore(IndexBase* owner, bool half)
      : ix(owner), d(owner->dim), s(owner->stream), want_mirror(half && d % 8 == 0), mirror(want_mirror) {}

  // grow to cap rows keeping the first `keep`.  Out of device memory drops the mirror, and the list scan streams the
  // FP32 rows instead.
  void grow(int64_t cap, int64_t keep) {
    vecs.reserve((size_t)cap * d, (size_t)keep * d, s);
    ids.reserve(cap, keep, s);
    norms.reserve(cap, keep, s);
    if (mirror && !(vecs_h.try_reserve((size_t)cap * d, (size_t)keep * d, s) && hscale.try_reserve(cap, keep, s))) {
      vecs_h.free(); hscale.free();
      mirror = false;
    }
  }
  // drop every row and buffer; the mirror is wanted again
  void reset() {
    vecs.free(); ids.free(); norms.free(); vecs_h.free(); hscale.free();
    mirror = want_mirror;
  }
  // copy rows [src, src + n) to [dst, dst + n) (list relocation)
  void move(int64_t src, int64_t dst, int64_t n) {
    B200VS_CUDA(cudaMemcpyAsync(vecs.p + (size_t)dst * d, vecs.p + (size_t)src * d, (size_t)n * d * 4, cudaMemcpyDeviceToDevice, s));
    B200VS_CUDA(cudaMemcpyAsync(ids.p + dst, ids.p + src, (size_t)n * 8, cudaMemcpyDeviceToDevice, s));
    B200VS_CUDA(cudaMemcpyAsync(norms.p + dst, norms.p + src, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
    if (mirror) {
      B200VS_CUDA(cudaMemcpyAsync(vecs_h.p + (size_t)dst * d, vecs_h.p + (size_t)src * d, (size_t)n * d * 2, cudaMemcpyDeviceToDevice, s));
      B200VS_CUDA(cudaMemcpyAsync(hscale.p + dst, hscale.p + src, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
    }
  }
  // x / xids: device rows and ids; row i goes to slot slots[i]
  void write(const float* x, const long long* xids, const std::vector<long long>& slots) {
    const int64_t n = (int64_t)slots.size();
    long long* d_slots = ix->scratch.alloc<long long>(n);
    float* row_norms = ix->scratch.alloc<float>(n);
    B200VS_CUDA(cudaMemcpyAsync(d_slots, slots.data(), (size_t)n * 8, cudaMemcpyHostToDevice, s));
    launch_scatter_rows(x, xids, d_slots, n, d, vecs.p, ids.p, norms.p, row_norms, s);
    if (mirror) launch_half_rows(vecs.p, d_slots, n, d, vecs_h.p, hscale.p, s);  // re-derived from the stored rows
    max_norm = std::max(max_norm, device_max_norm(ix, row_norms, n, s));
  }
  // compaction: fresh buffers of cap rows holding row src[i] at dst[i].  The mirror is re-derived from the moved FP32
  // rows, which gives the same bits as moving the old mirror rows.
  void gather(const std::vector<long long>& src, const std::vector<long long>& dst, int64_t cap) {
    const int64_t n = (int64_t)src.size();
    DevBuf<float> nv; DevBuf<long long> ni; DevBuf<float> nn;
    nv.reserve((size_t)cap * d, 0, s); ni.reserve(cap, 0, s); nn.reserve(cap, 0, s);
    long long* d_dst = nullptr;
    if (n) {
      long long* d_src = ix->scratch.alloc<long long>(n);
      d_dst = ix->scratch.alloc<long long>(n);
      B200VS_CUDA(cudaMemcpyAsync(d_src, src.data(), n * 8, cudaMemcpyHostToDevice, s));
      B200VS_CUDA(cudaMemcpyAsync(d_dst, dst.data(), n * 8, cudaMemcpyHostToDevice, s));
      launch_move_rows(vecs.p, ids.p, norms.p, d_src, d_dst, n, d, nv.p, ni.p, nn.p, s);
    }
    B200VS_CUDA(cudaStreamSynchronize(s));
    vecs.swap(nv); ids.swap(ni); norms.swap(nn);
    if (mirror) {
      vecs_h.free(); hscale.free();
      grow(cap, 0);  // the FP32 arrays already hold cap rows: allocates the mirror only
      if (mirror && n) launch_half_rows(vecs.p, d_dst, n, d, vecs_h.p, hscale.p, s);
    }
  }
  // rows [r0, r0 + n) as FP32 rows [n, d] on the host
  size_t row_bytes() const { return (size_t)d * 4; }
  void download(int64_t r0, int64_t n, uint8_t* out) const {
    if (n > 0) B200VS_CUDA(cudaMemcpy(out, vecs.p + (size_t)r0 * d, (size_t)n * d * 4, cudaMemcpyDeviceToHost));
  }
  const void* row_data() const { return vecs.p; }
  size_t row_pitch() const { return (size_t)d * 4; }
  int64_t bytes() const { return (int64_t)(vecs.cap * 4 + ids.cap * 8 + norms.cap * 4 + vecs_h.cap * 2 + hscale.cap * 4); }
  // the row fields of a tile-scan view; the owner adds the list layout
  TcView view() const {
    TcView v;
    v.vecs = vecs.p; v.ids = ids.p; v.norms = norms.p; v.max_norm = max_norm;
    if (mirror) { v.vecs_h = vecs_h.p; v.hscale = hscale.p; }
    return v;
  }
};

// ============================================================================================
// Flat
// ============================================================================================
struct FlatIndex : IndexBase {
  FlatRowMap<RowStore> rowmap{this, false};  // no mirror: a Flat search keeps its TF32 arithmetic

  FlatIndex(b200vs_metric m, int d, const b200vs_params& p) : IndexBase(B200VS_FLAT, m, d, p) {}

  // VectorIndexFlat::AddOrUpsert, vector_index_flat.cc:121-162: duplicate ids inside the batch are rejected,
  // pre-existing ids are ALWAYS removed first (add and upsert behave the same), then add_with_ids.  Device rows come from
  // the owner of a row-sharded add, a snapshot restore and a rebuild.
  void add(const AddReq& r) override {
    if (r.ids) check_batch_ids_unique(r.n, r.ids);
    WriteHold hold(this);
    const bool normalise = metric == B200VS_COSINE && r.form == AddReq::RAW;  // the normaliser works in place
    Staged st;
    stage(r, (size_t)dim * 4, normalise, st);
    if (!r.ids) check_batch_ids_unique(r.n, st.ids);
    if (normalise) launch_normalize_faiss(static_cast<float*>(st.x), r.n, dim, stream);  // flat.cc:155 (normalize_)
    rowmap.add(r.n, static_cast<const float*>(st.x), st.ids_dev, st.ids);
  }

  void check_add(const AddReq& r) override { IndexBase::check_add(r); check_batch_ids_unique(r.n, r.ids); }

  // streaming brute-force scan (b200vs_scan_*): the tile index is emptied between tiles, buffers are kept
  void clear() override {
    WriteHold hold(this);
    rowmap.store.max_norm = 0.f;
    rowmap.clear();
  }

  // VectorIndexFlat::Delete, vector_index_flat.cc:171-203: unknown ids are ignored (only ids present in
  // rev_map are handed to remove_ids).
  int64_t remove(int64_t n, const int64_t* del) override {
    WriteHold hold(this);
    return rowmap.remove(n, del);
  }

  ScanJob job(const SearchCtx& sc) const {
    ScanJob j;
    j.l2 = metric == B200VS_L2;
    j.vecs = rowmap.store.vecs.p; j.ids = rowmap.store.ids.p; j.d = dim; j.mode = 0; j.n = rowmap.rows; j.sc = &sc;
    return j;
  }

  // VectorIndexFlat::Search / RangeSearch, vector_index_flat.cc:206-323
  void search(const SearchReq& r, cudaStream_t s) override {
    refuse_probes(r);
    flat_view_search(this, rowmap.view(), r, s);
  }

  // the store's ids already mark every tombstone
  bool brute_force_rows(TcView& v, bool, cudaStream_t) override {
    v = rowmap.view();
    return rowmap.rows > 0;
  }

  void debug_tc_scores(int64_t nq, const float* xq, int arith, float* out_scores, float* out_eps, cudaStream_t s) override {
    const int64_t rows = rowmap.rows;
    if ((double)nq * (double)rows * 4 > (double)(1LL << 30)) fail(B200VS_EILLEGAL_PARAMETERS, "score matrix larger than 1 GiB");
    const float* q = prepare_queries(nq, xq, s);
    float* ds = scratch.alloc<float>((size_t)std::max<int64_t>(nq * rows, 1));
    float* de = scratch.alloc<float>(nq);
    const bool sample = arith >= 3;  // 3 / 4: the sample pass in the TF32 / FP16 list-scan arithmetic
    const TcArith a = sample ? (arith == 4 ? TC_ARITH_FP16 : TC_ARITH_TF32) : (TcArith)arith;
    tc_debug_scores(this, rowmap.view(), metric == B200VS_L2, nq, q, a, sample, ds, de, s);
    if (rows > 0) B200VS_CUDA(cudaMemcpyAsync(out_scores, ds, (size_t)nq * rows * 4, cudaMemcpyDeviceToHost, s));
    B200VS_CUDA(cudaMemcpyAsync(out_eps, de, (size_t)nq * 4, cudaMemcpyDeviceToHost, s));
    B200VS_CUDA(cudaStreamSynchronize(s));
  }

  void reconstruct(int64_t n, const int64_t* in_ids, float* out, uint8_t* found) override {
    RwSharedGuard rl(this);
    std::lock_guard<std::mutex> gl(gpu_mu);
    set_device();
    for (int64_t i = 0; i < n; ++i) {
      auto it = rowmap.id2row.find(in_ids[i]);
      if (found) found[i] = it != rowmap.id2row.end() ? 1 : 0;
      if (it != rowmap.id2row.end())
        B200VS_CUDA(cudaMemcpyAsync(out + (size_t)i * dim, rowmap.store.vecs.p + (size_t)it->second * dim, (size_t)dim * 4, cudaMemcpyDeviceToHost, stream));
    }
    B200VS_CUDA(cudaStreamSynchronize(stream));
  }
  int64_t count() const override { return rowmap.count(); }
  int64_t deleted_count() const override { return rowmap.ndeleted; }
  int64_t memory_size() const override { return rowmap.store.bytes(); }
  void live_rows(int64_t lo, int64_t hi, RebuildSource& out) override {
    rowmap.live_slots(out.ids, out.slots, lo, hi);
    out.rows = reinterpret_cast<const uint32_t*>(rowmap.store.vecs.p);
    out.stream = stream;
  }
  // the sources' stored rows in ascending id order in one add (cosine rows are already normalised)
  int64_t rebuild_from(const std::vector<IndexBase*>& srcs, int64_t lo, int64_t hi) override {
    DevBuf<uint32_t> rows;
    DevBuf<long long> ids;
    const int64_t n = sorted_live_rows(this, srcs, lo, hi, dim, rows, ids, stream);
    if (n == 0) return 0;
    std::vector<int64_t> h_ids(n);
    B200VS_CUDA(cudaMemcpyAsync(h_ids.data(), ids.p, (size_t)n * 8, cudaMemcpyDeviceToHost, stream));
    B200VS_CUDA(cudaStreamSynchronize(stream));
    rowmap.add(n, reinterpret_cast<const float*>(rows.p), ids.p, h_ids.data());
    return n;
  }

  void export_lists(int64_t* list_off, float* vectors, uint8_t*, int64_t* out_ids) override {
    RwSharedGuard rl(this);
    std::lock_guard<std::mutex> gl(gpu_mu);
    set_device();
    quiesce();
    rowmap.export_rows(list_off, reinterpret_cast<uint8_t*>(vectors), out_ids);
  }
  void pack_lists(int64_t* list_off, void* out_ids, uint8_t* out_rows) override {
    RwSharedGuard rl(this);
    std::lock_guard<std::mutex> gl(gpu_mu);
    set_device();
    quiesce();
    rowmap.pack(list_off, out_ids, out_rows);
  }
};

IndexBase* make_flat(b200vs_metric m, int d, const b200vs_params& p) { return new FlatIndex(m, d, p); }

// range radius -> 1 - radius for IP / cosine (vector_index_flat.cc:282-285); faiss range_search keeps L2 dis < radius, IP
// ip > radius.  Every path selects the same rows.
void flat_view_search(IndexBase* ix, const TcView& v, const SearchReq& r, cudaStream_t s) {
  const float* q = ix->queries(r, s);
  const float thr = ix->ip_like() ? 1.0F - r.radius : r.radius;
  ScanJob j;
  j.l2 = ix->metric == B200VS_L2;
  j.vecs = v.vecs; j.ids = v.ids; j.d = ix->dim; j.mode = 0; j.n = v.arena_rows; j.sc = r.sc;
  if (r.deep) { run_scan_deep(ix, j, r.nq, q, r.k, r.od, r.raw, r.oi, s); return; }
  if (v.arena_rows > 0 && tc_eligible(ix, v, r.nq, r.k, 1, *r.sc, r.range)) {
    long long* probes = ix->scratch.alloc<long long>(r.nq);
    B200VS_CUDA(cudaMemsetAsync(probes, 0, (size_t)r.nq * 8, s));
    tc_search(ix, v, r, q, probes, 1, thr, s);
    return;
  }
  if (!r.range && flat_small_eligible(ix->device, r.nq, v.arena_rows, ix->dim, r.k, *r.sc)) {  // one query per task is the reference's own shape: single-launch path
    flat_small_search(ix, j.l2, v.vecs, v.ids, v.arena_rows, r.nq, q, r.k, *r.sc, r.od, r.oi, r.raw, s);
    return;
  }
  if (r.range) { j.has_thr = true; j.thr_raw = thr; }
  run_scan(ix, j, r.nq, q, r.k, r.raw ? nullptr : r.od, r.raw ? r.od : nullptr, r.oi, r.oc, s);
}

// ============================================================================================
// IVF-Flat
// ============================================================================================

void fill_empty(const SearchReq& r, cudaStream_t s) {
  if (r.od) B200VS_CUDA(cudaMemsetAsync(r.od, 0, (size_t)r.nq * r.k * 4, s));
  B200VS_CUDA(cudaMemsetAsync(r.oi, 0xFF, (size_t)r.nq * r.k * 8, s));  // -1
  if (r.range && r.oc) B200VS_CUDA(cudaMemsetAsync(r.oc, 0, (size_t)r.nq * 4, s));
}

struct IvfFlatIndex : IndexBase {
  int nlist;            // may degenerate to 1 at train time (vector_index_ivf_flat.cc:676-680)
  bool trained = false;
  DevBuf<float> centroids;       // [nlist, d]
  DevBuf<long long> cent_ids;    // iota
  DevBuf<float> cent_norms;      // ||c||^2 (tensor-core coarse pass)
  RowStore store{this, true};    // the arena, [L.arena_cap] rows, with the FP16 mirror the list scan streams
  IvfLists L;                    // host bookkeeping + device list_off/list_len
  float cent_max_norm = 0.f;
  DevBuf<float> cent_hi, cent_lo;  // error-compensated split of the centroids (tc_coarse)
  DevBuf<long long> d_coff;  // the centroid table seen as one "list" by the tensor-core coarse pass
  // Centroid rows [c0, c0 + rows) of a centroid table (the installed one, or k-means' current one), with its error-compensated
  // split and norms, as the one list tc_coarse scans; the rows it returns are numbered from c0.
  TcView coarse_view(const float* vecs, const float* hi, const float* lo, const float* norms, float max_norm, int c0, int rows) const {
    TcView v;
    v.vecs = vecs + (size_t)c0 * dim; v.vecs_hi = hi + (size_t)c0 * dim; v.vecs_lo = lo + (size_t)c0 * dim;
    v.ids = cent_ids.p + c0; v.norms = norms + c0; v.max_norm = max_norm; v.id_offset = c0;
    v.arena_rows = rows; v.list_off = d_coff.p;
    v.nlist = 1; v.flat = true; v.total_chunks = (rows + TC_CHUNK - 1) / TC_CHUNK; v.max_chunks_per_list = (int)v.total_chunks;
    return v;
  }
  TcView view() const {
    TcView v = store.view();
    v.arena_rows = L.arena_used; v.list_off = L.d_off.p; v.list_len = L.d_len.p;
    v.nlist = nlist; v.total_chunks = L.total_chunks; v.max_chunks_per_list = L.max_chunks_per_list;
    return v;
  }

  IvfFlatIndex(b200vs_metric m, int d, const b200vs_params& p) : IndexBase(B200VS_IVF_FLAT, m, d, p) {
    nlist = p.nlist > 0 ? p.nlist : 2048;  // Constant::kCreateIvfFlatParamNcentroids
  }
  bool is_trained() const override { return trained; }
  int export_nlist() const override { return nlist; }

  void install_centroids(const float* host_c, int k) {
    quiesce();
    nlist = k;
    centroids.free(); cent_ids.free(); cent_norms.free();
    centroids.reserve((size_t)k * dim, 0, stream);
    cent_ids.reserve(k, 0, stream);
    cent_norms.reserve(k, 0, stream);
    B200VS_CUDA(cudaMemcpyAsync(centroids.p, host_c, (size_t)k * dim * 4, cudaMemcpyHostToDevice, stream));
    launch_iota(cent_ids.p, k, stream);
    launch_row_norms(centroids.p, k, dim, cent_norms.p, stream);
    cent_hi.free(); cent_lo.free();
    cent_hi.reserve((size_t)k * dim, 0, stream); cent_lo.reserve((size_t)k * dim, 0, stream);
    launch_split_rows(centroids.p, k, dim, cent_hi.p, cent_lo.p, stream);
    cent_max_norm = device_max_norm(this, cent_norms.p, k, stream);
    d_coff.reserve(1, 0, stream);
    B200VS_CUDA(cudaMemsetAsync(d_coff.p, 0, 8, stream));
    B200VS_CUDA(cudaStreamSynchronize(stream));
    L.init(k, stream);
    store.reset();
    trained = true;
  }

  // trained-state blob: int64 hdr[4] = {magic 'IVFC', nlist, dim, metric}; float centroids[nlist*dim]
  static constexpr int64_t kStateMagic = 0x43465649;
  void state_header(void* blob, int k) const {
    const int64_t hdr[4] = {kStateMagic, k, dim, (int64_t)metric};
    memcpy(blob, hdr, 32);
  }
  void set_state(const void* blob, size_t len) override {
    WriteHold hold(this);
    if (len < 32) fail(B200VS_EILLEGAL_PARAMETERS, "state blob too short");
    const int64_t* hdr = (const int64_t*)blob;
    if (hdr[0] != kStateMagic || hdr[2] != dim) fail(B200VS_EILLEGAL_PARAMETERS, "bad IVF state blob");
    const int k = (int)hdr[1];
    if (len < 32 + (size_t)k * dim * 4) fail(B200VS_EILLEGAL_PARAMETERS, "state blob truncated");
    install_centroids((const float*)((const char*)blob + 32), k);
  }
  int64_t get_state(void* blob, size_t cap) override {
    RwSharedGuard rl(this);
    if (!trained) return 0;
    const size_t need = 32 + (size_t)nlist * dim * 4;
    if (!blob || cap < need) return (int64_t)need;
    set_device();
    state_header(blob, nlist);
    B200VS_CUDA(cudaMemcpyAsync((char*)blob + 32, centroids.p, (size_t)nlist * dim * 4, cudaMemcpyDeviceToHost, stream));
    B200VS_CUDA(cudaStreamSynchronize(stream));
    return (int64_t)need;
  }

  // assign rows (device, already normalised) to their nearest centroid: IndexFlat quantiser, k = 1.  Large batches go
  // through the tensor-core coarse pass (certified exact, so the labels equal the exact scan's).
  void assign_dev(const float* x_dev, int64_t n, long long* out_list_dev, cudaStream_t s) {
    const int64_t chunk = std::max<int64_t>(1024, std::min<int64_t>(32768, (1LL << 28) / std::max(1, nlist)));
    for (int64_t a = 0; a < n; a += chunk) {
      const int64_t m = std::min(chunk, n - a);
      const auto mark = scratch.mark();
      coarse_rows(m, x_dev + (size_t)a * dim, 1, 0, nlist, true, nullptr, out_list_dev + a, s);
      scratch.release(mark);  // stream-ordered reuse
    }
  }

  // VectorIndexIvfFlat::Train, vector_index_ivf_flat.cc:644-712 -> faiss IndexIVFFlat::train ->
  // Clustering (niter 10, seed 1234, <= 256 points per centroid); GPU Lloyd iterations here.
  void train(int64_t n, const void* x) override;
  // train's rule with rw and gpu_mu held: x on the host (raw), or on the device (x_dev: already prepared)
  void train_locked(int64_t n, const float* x, bool x_dev);

  // VectorIndexIvfFlat::NeedToRebuild, vector_index_ivf_flat.cc:751-776 (max_points_per_centroid = 256)
  bool need_rebuild() const override {
    if (!trained) return false;
    const int64_t nlist_org = params.nlist > 0 ? params.nlist : 2048;
    if (nlist == nlist_org && nlist == 1) return false;
    if (nlist != nlist_org && nlist == 1 && L.live >= 256 * nlist_org) return true;
    if (nlist == nlist_org && nlist != 1 && L.live >= 256 * nlist_org) return train_rows <= L.live / 2;
    return false;
  }
  void live_rows(int64_t lo, int64_t hi, RebuildSource& out) override {
    L.live_slots(out.ids, out.slots, lo, hi);
    out.rows = reinterpret_cast<const uint32_t*>(store.vecs.p);
    out.stream = stream;
  }
  // train on the sources' stored rows in ascending id order, then add them in that order; stored cosine rows are already
  // normalised
  int64_t rebuild_from(const std::vector<IndexBase*>& srcs, int64_t lo, int64_t hi) override {
    DevBuf<uint32_t> rows;
    DevBuf<long long> ids;
    const int64_t n = sorted_live_rows(this, srcs, lo, hi, dim, rows, ids, stream);
    if (n == 0) return 0;
    train_locked(n, reinterpret_cast<const float*>(rows.p), true);
    scratch.reset(stream);
    add_locked(AddReq::device(n, rows.p, ids.p, nullptr, false, AddReq::PREPARED));
    return n;
  }

  void add(const AddReq& r) override;
  void add_locked(const AddReq& r);
  void reserve_lists(const int64_t* rows_per_list, int n_lists) override;
  int nlist_now() const override { return nlist; }
  void assign_lists_dev(int64_t n, const void* x_dev, long long* out_lists_dev, cudaStream_t s) override {
    if (!trained) fail(B200VS_EVECTOR_NOT_TRAIN, "not train");
    assign_dev(static_cast<const float*>(x_dev), n, out_lists_dev, s);
  }
  int resolve_nprobe_api(const SearchCtx& sc) const override { return resolve_nprobe(sc); }
  int64_t remove(int64_t n, const int64_t* del) override;

  int resolve_nprobe(const SearchCtx& sc) const {
    int np = sc.nprobe > 0 ? sc.nprobe : 80;  // Constant::kSearchIvfFlatParamNprobe, ivf_flat.cc:211
    return std::min(np, nlist);               // ivf_flat.cc:234
  }

  void search(const SearchReq& r, cudaStream_t s) override;
  // the arena with its FP16 mirror; the ids of the slots outside every list's [off, off + len) (capacity slack, the old
  // places of relocated lists) are -1 in a view built per call
  bool brute_force_rows(TcView& v, bool, cudaStream_t s) override {
    if (!trained || L.live == 0) return false;
    v = store.view();
    const int64_t rows = L.arena_used;
    long long* ids = scratch.alloc<long long>(rows);
    launch_list_ids(store.ids.p, L.d_off.p, L.d_len.p, nlist, rows, ids, s);
    launch_count(1);
    v.ids = ids;
    long long* off = scratch.alloc<long long>(1);
    int* len = scratch.alloc<int>(1);
    const int len1 = (int)std::min<int64_t>(rows, 0x7fffffff);
    B200VS_CUDA(cudaMemsetAsync(off, 0, 8, s));
    B200VS_CUDA(cudaMemcpyAsync(len, &len1, 4, cudaMemcpyHostToDevice, s));
    set_flat_layout(v, rows, off, len);
    return true;
  }
  void coarse(int64_t nq, const void* xv, bool prepared, int nprobe, int c0, int c1, float* out_score, long long* out_lists,
              cudaStream_t s) override {
    if (!trained) fail(B200VS_EVECTOR_NOT_TRAIN, "not train");
    if (c0 < 0 || c1 > nlist || c0 >= c1 || nprobe <= 0 || nprobe > c1 - c0) fail(B200VS_EILLEGAL_PARAMETERS, "bad centroid range / nprobe");
    const float* xq = static_cast<const float*>(xv);
    coarse_rows(nq, prepared ? xq : prepare_queries(nq, xq, s), nprobe, c0, c1, true, out_score, out_lists, s);
  }

  // the nprobe nearest of centroid rows [c0, c1) of prepared queries: the tensor-core pass (dense TF32 scores + certified
  // exact re-score) when allowed and the shapes fit, else the exact scan.  out_score: coarse's ascending ranking score.
  void coarse_rows(int64_t nq, const float* q, int nprobe, int c0, int c1, bool allow_tc, float* out_score, long long* out_lists,
                   cudaStream_t s) {
    const int rows = c1 - c0;
    if (allow_tc && tc_coarse_eligible(this, nq, rows, nprobe) && tc_norms_in_range(metric == B200VS_L2, cent_max_norm)) {
      TcView v = coarse_view(centroids.p, cent_hi.p, cent_lo.p, cent_norms.p, cent_max_norm, c0, rows);
      v.api_scores = out_score != nullptr;
      tc_coarse(this, v, metric == B200VS_L2, nq, q, nprobe, out_lists, out_score, s);
      return;
    }
    ScanJob j;
    j.l2 = metric == B200VS_L2;
    j.vecs = centroids.p + (size_t)c0 * dim; j.ids = cent_ids.p + c0; j.d = dim; j.mode = 0; j.n = rows;
    run_scan(this, j, nq, q, nprobe, nullptr, out_score, out_lists, nullptr, s);          // raw metric value
    if (out_score && metric != B200VS_L2) launch_negate(out_score, nq * nprobe, s);   // -> ascending ranking score
  }
  ScanJob list_job(const SearchCtx& sc, const long long* probes, int nprobe) const {
    ScanJob j;
    j.l2 = metric == B200VS_L2;
    j.vecs = store.vecs.p; j.ids = store.ids.p; j.d = dim; j.mode = 1; j.probes = probes; j.nprobe = nprobe;
    j.list_off = L.d_off.p; j.list_len = L.d_len.p; j.sc = &sc;
    j.avg_candidates = nlist > 0 ? (double)L.total_len() * nprobe / nlist : 0;
    return j;
  }

  int64_t count() const override { return L.live; }
  int64_t deleted_count() const override { return L.dead; }
  int64_t memory_size() const override {
    return store.bytes() + (int64_t)centroids.cap * 4;
  }
  void export_lists(int64_t* list_off, float* vectors, uint8_t*, int64_t* out_ids) override;
  int64_t export_list(int list, int64_t cap, float* vectors, int64_t* out_ids) override;
  void pack_lists(int64_t* list_off, void* out_ids, uint8_t* out_rows) override {
    RwSharedGuard rl(this);
    std::lock_guard<std::mutex> gl(gpu_mu);
    set_device();
    quiesce();
    L.pack(nlist, list_off, store, out_ids, out_rows);
  }
};

void IvfFlatIndex::train(int64_t n, const void* x) {
  if (n <= 0) fail(B200VS_EILLEGAL_PARAMETERS, "data size invalid");
  WriteHold hold(this);
  if (trained) return;  // ivf_flat.cc:670-672
  train_locked(n, static_cast<const float*>(x), false);
}

void IvfFlatIndex::train_locked(int64_t n, const float* x, bool x_dev) {
  int k = nlist;
  if (n < k) k = 1;  // "data size too small, nlist degenerate to 1", ivf_flat.cc:676-680
  std::vector<float> cent;
  auto assign = [&](const float* xd, int64_t m, const float* cd, int kk, long long* out) {
    // assignment against the CURRENT centroids cd (device): tensor-core coarse pass when the shapes allow (certified
    // exact labels), else the exact scan
    const int64_t chunk = std::max<int64_t>(1024, std::min<int64_t>(32768, (1LL << 28) / std::max(1, kk)));
    const auto mark0 = scratch.mark();
    TcView cv;
    const bool use_tc = tc_coarse_eligible(this, std::min(chunk, m), kk, 1);
    if (use_tc) {
      float* hi = scratch.alloc<float>((size_t)kk * dim);
      float* lo = scratch.alloc<float>((size_t)kk * dim);
      float* nr = scratch.alloc<float>(kk);
      launch_split_rows(cd, kk, dim, hi, lo, stream);
      launch_row_norms(cd, kk, dim, nr, stream);
      cv = coarse_view(cd, hi, lo, nr, device_max_norm(this, nr, kk, stream), 0, kk);
    }
    ScanJob j;
    j.l2 = metric == B200VS_L2;
    j.vecs = cd; j.ids = cent_ids.p; j.d = dim; j.mode = 0; j.n = kk;
    for (int64_t a = 0; a < m; a += chunk) {
      const int64_t mm = std::min(chunk, m - a);
      const auto mark = scratch.mark();
      if (use_tc && mm >= 16) tc_coarse(this, cv, metric == B200VS_L2, mm, xd + (size_t)a * dim, 1, out + a, nullptr, stream);
      else run_scan(this, j, mm, xd + (size_t)a * dim, 1, nullptr, nullptr, out + a, nullptr, stream);
      scratch.release(mark);
    }
    scratch.release(mark0);
  };
  auto prepare_ids = [&](int kk) {
    cent_ids.free(); cent_ids.reserve(kk, 0, stream); launch_iota(cent_ids.p, kk, stream);
    d_coff.reserve(1, 0, stream);
    B200VS_CUDA(cudaMemsetAsync(d_coff.p, 0, 8, stream));
  };
  if (x_dev) kmeans_gpu_dev(this, dim, n, x, k, 10, 256, 1234, cent, assign, prepare_ids);
  else kmeans_gpu(this, metric, dim, n, x, k, 10, 256, 1234, cent, assign, prepare_ids);
  install_centroids(cent.data(), k);
  train_rows = n;
}

// untrained -> refused (ivf_flat.cc:111-113; the caller trains and retries, :136-150); upsert removes the ids first (:115-118)
void IvfFlatIndex::add(const AddReq& r) {
  WriteHold hold(this);
  if (!trained) fail(B200VS_EVECTOR_NOT_TRAIN, "not train");
  add_locked(r);
}

// add with the writer hold taken
void IvfFlatIndex::add_locked(const AddReq& r) {
  const bool normalise = metric == B200VS_COSINE && r.form == AddReq::RAW;  // the normaliser works in place
  Staged st;
  stage(r, (size_t)dim * 4, normalise, st);
  float* x = static_cast<float*>(st.x);
  if (normalise) launch_normalize_faiss(x, r.n, dim, stream);
  std::vector<long long> h_list;
  IvfLists::row_lists(this, r.n, r.lists, h_list, [&](long long* out) { assign_dev(x, r.n, out, stream); });
  L.place(r.n, h_list.data(), st.ids, x, st.ids_dev, store, r.upsert);
}

void IvfFlatIndex::reserve_lists(const int64_t* rows_per_list, int n_lists) {
  WriteHold hold(this);
  if (!trained) fail(B200VS_EVECTOR_NOT_TRAIN, "not train");
  L.reserve(rows_per_list, n_lists, store);
}

// VectorIndexIvfFlat::Delete, vector_index_ivf_flat.cc:162-189: untrained -> OK; nothing removed -> EVECTOR_INVALID.
int64_t IvfFlatIndex::remove(int64_t n, const int64_t* del) {
  WriteHold hold(this);
  if (!trained) return -1;  // signalled as OK by the ABI
  return L.remove(n, del, store);
}

// VectorIndexIvfFlat::Search / RangeSearch, vector_index_ivf_flat.cc:203-350: untrained -> empty results (:224-227); range
// radius -> 1 - radius for IP / cosine (:296-299).  The index's own coarse pass keeps to exact_only for top-k only.
void IvfFlatIndex::search(const SearchReq& r, cudaStream_t s) {
  if (!trained) { fill_empty(r, s); return; }
  const SearchCtx& sc = *r.sc;
  const float* q = queries(r, s);
  const int nprobe = r.probes ? r.nprobe : resolve_nprobe(sc);
  const long long* probes = r.probes;
  if (!probes) {
    long long* own = scratch.alloc<long long>((size_t)r.nq * nprobe);
    coarse_rows(r.nq, q, nprobe, 0, nlist, r.range || !sc.exact_only, nullptr, own, s);
    probes = own;
  }
  if (profiling) profile_probed(this, probes, r.nq * nprobe, nlist, L.d_len.p, s);
  if (r.deep) { run_scan_deep(this, list_job(sc, probes, nprobe), r.nq, q, r.k, r.od, r.raw, r.oi, s); return; }
  const float thr = ip_like() ? 1.0F - r.radius : r.radius;
  const TcView v = view();
  if (L.live > 0 && tc_eligible(this, v, r.nq, r.k, nprobe, sc, r.range)) {
    tc_search(this, v, r, q, probes, nprobe, thr, s);
    return;
  }
  ScanJob j = list_job(sc, probes, nprobe);
  if (r.range) { j.has_thr = true; j.thr_raw = thr; }
  else j.dominant = true;
  run_scan(this, j, r.nq, q, r.k, r.raw ? nullptr : r.od, r.raw ? r.od : nullptr, r.oi, r.oc, s);
}

void IvfFlatIndex::export_lists(int64_t* list_off, float* vectors, uint8_t*, int64_t* out_ids) {
  RwSharedGuard rl(this);
  std::lock_guard<std::mutex> gl(gpu_mu);
  set_device();
  quiesce();
  L.export_lists(nlist, list_off, store, reinterpret_cast<uint8_t*>(vectors), out_ids);
}

int64_t IvfFlatIndex::export_list(int list, int64_t cap, float* vectors, int64_t* out_ids) {
  RwSharedGuard rl(this);
  std::lock_guard<std::mutex> gl(gpu_mu);
  if (list < 0 || list >= nlist) fail(B200VS_EILLEGAL_PARAMETERS, "list id out of range");
  set_device();
  quiesce();
  return L.export_list(list, cap, store, reinterpret_cast<uint8_t*>(vectors), out_ids);
}

IndexBase* make_ivf_flat(b200vs_metric m, int d, const b200vs_params& p) { return new IvfFlatIndex(m, d, p); }

static IvfFlatIndex* as_ivf_flat(IndexBase* ix) {
  auto* p = dynamic_cast<IvfFlatIndex*>(ix);
  if (!p) fail(B200VS_EINTERNAL, "not an IVF_FLAT index");
  return p;
}

void ivf_flat_train_coarse(IndexBase* ix, int64_t n, const float* x, bool x_dev, int k, std::vector<float>& cent) {
  b200vs_params p = as_ivf_flat(ix)->params;
  p.nlist = k;
  IvfFlatIndex loc(ix->metric, ix->dim, p);  // train on an index of its own: ix keeps its state and lists
  if (x_dev) {
    WriteHold hold(&loc);
    loc.train_locked(n, x, true);
  } else {
    loc.train(n, x);
  }
  cent.resize((size_t)loc.nlist * loc.dim);
  B200VS_CUDA(cudaMemcpy(cent.data(), loc.centroids.p, cent.size() * 4, cudaMemcpyDeviceToHost));
}

void ivf_flat_train_state(IndexBase* ix, const std::vector<float>& cent, std::vector<unsigned char>& blob) {
  const IvfFlatIndex* f = as_ivf_flat(ix);
  blob.resize(32 + cent.size() * 4);
  f->state_header(blob.data(), (int)(cent.size() / f->dim));
  memcpy(blob.data() + 32, cent.data(), cent.size() * 4);
}

}  // namespace b200vs
