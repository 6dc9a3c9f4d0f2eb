// binary.cu — Binary Flat and Binary IVF-Flat: Hamming search over packed bits.
//
// The GPU replacements of the faiss::IndexBinary instantiations of the Flat and IVF-Flat plugins
// (VectorIndexFlat<IndexBinary, IndexBinaryIDMap2>, src/vector/vector_index_flat.cc:71, :99-102;
// VectorIndexIvfFlat<IndexBinary>, vector_index_ivf_flat.cc:62; built by vector_index_factory.cc:73-80, :381-425).
//
// Rows are packed bits, dim / 8 bytes each.  On the device a row takes w = ceil(dim / 32) 32-bit words, zero padded, and
// queries are padded the same way, so the padding adds 0 to every XOR popcount.  Batches with enough work (bt_eligible)
// run on the BMMA tile scan (binary_tile.cu); the rest, range searches and the coarse quantiser run on the exact scan
// (scan_select_kernel<HammingDist> + merge_select_kernel, scan_kernels.cuh).  Both use the key f2ord((float)distance):
// distances are exact integers <= 32768, so the key orders them like the integers and results are ordered by
// (distance, id), identical on both paths.
#include <cmath>

#include "binary_tile.cuh"
#include "index.h"
#include "ivf_common.h"

namespace b200vs {

namespace {

// dst[r, j] = bytes 4j .. 4j+3 of packed row r (little-endian word), zero past nbytes
__global__ void pad_rows_kernel(const uint8_t* __restrict__ src, long long n, int nbytes, int w, uint32_t* __restrict__ dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * w) return;
  const long long r = i / w;
  const int j = (int)(i % w);
  const uint8_t* row = src + (size_t)r * nbytes;
  uint32_t v = 0;
  for (int b = 0; b < 4; ++b)
    if (4 * j + b < nbytes) v |= (uint32_t)row[4 * j + b] << (8 * b);
  dst[i] = v;
}

// dst row dst_rows[r] = src row (src_rows ? src_rows[r] : r), words and id
__global__ void copy_rows_kernel(const uint32_t* __restrict__ src, const long long* __restrict__ sids, const long long* __restrict__ src_rows,
                                 const long long* __restrict__ dst_rows, long long n, int w, uint32_t* dst, long long* dids) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * w) return;
  const long long r = i / w;
  const int j = (int)(i % w);
  const long long sr = src_rows ? src_rows[r] : r, dr = dst_rows[r];
  dst[(size_t)dr * w + j] = src[(size_t)sr * w + j];
  if (j == 0) dids[dr] = sids[sr];
}

int words_of(int dim) { return (dim / 8 + 3) / 4; }

}  // namespace

void launch_pad_rows(const uint8_t* src, int64_t n, int nbytes, uint32_t* dst, cudaStream_t s) {
  const int w = (nbytes + 3) / 4;
  if (n <= 0) return;
  pad_rows_kernel<<<(unsigned)cdiv(n * w, 256), 256, 0, s>>>(src, n, nbytes, w, dst);
  B200VS_CUDA(cudaGetLastError());
}

// Device rows of a binary index: [cap, w] words and ids (-1 = tombstone / unused slot).  The owner decides capacities and
// slots; the store moves rows.  All work runs on the owner's stream.
struct BinRows {
  IndexBase* const ix;
  const int w;
  DevBuf<uint32_t> words;
  DevBuf<long long> ids;
  explicit BinRows(IndexBase* owner) : ix(owner), w(words_of(owner->dim)) {}

  void grow(int64_t cap, int64_t keep) {
    words.reserve((size_t)cap * w, (size_t)keep * w, ix->stream);
    ids.reserve(cap, keep, ix->stream);
  }
  void reset() { words.free(); ids.free(); }
  void move(int64_t src, int64_t dst, int64_t n) {
    B200VS_CUDA(cudaMemcpyAsync(words.p + (size_t)dst * w, words.p + (size_t)src * w, (size_t)n * w * 4, cudaMemcpyDeviceToDevice, ix->stream));
    B200VS_CUDA(cudaMemcpyAsync(ids.p + dst, ids.p + src, (size_t)n * 8, cudaMemcpyDeviceToDevice, ix->stream));
  }
  void copy(const uint32_t* src, const long long* sids, const long long* src_rows, const long long* dst_rows, int64_t n, uint32_t* dst,
            long long* dids) {
    if (n <= 0) return;
    copy_rows_kernel<<<(unsigned)cdiv(n * w, 256), 256, 0, ix->stream>>>(src, sids, src_rows, dst_rows, n, w, dst, dids);
    B200VS_CUDA(cudaGetLastError());
  }
  // x / xids: device padded rows and ids; row i goes to slot slots[i]
  void write(const uint32_t* x, const long long* xids, const std::vector<long long>& slots) {
    const int64_t n = (int64_t)slots.size();
    long long* d_slots = ix->scratch.alloc<long long>(n);
    B200VS_CUDA(cudaMemcpyAsync(d_slots, slots.data(), (size_t)n * 8, cudaMemcpyHostToDevice, ix->stream));
    copy(x, xids, nullptr, d_slots, n, words.p, ids.p);
  }
  // compaction: fresh buffers of cap rows holding row src[i] at dst[i]
  void gather(const std::vector<long long>& src, const std::vector<long long>& dst, int64_t cap) {
    const int64_t n = (int64_t)src.size();
    DevBuf<uint32_t> nw; DevBuf<long long> ni;
    nw.reserve((size_t)cap * w, 0, ix->stream); ni.reserve(cap, 0, ix->stream);
    if (n) {
      long long* d_src = ix->scratch.alloc<long long>(n);
      long long* d_dst = ix->scratch.alloc<long long>(n);
      B200VS_CUDA(cudaMemcpyAsync(d_src, src.data(), n * 8, cudaMemcpyHostToDevice, ix->stream));
      B200VS_CUDA(cudaMemcpyAsync(d_dst, dst.data(), n * 8, cudaMemcpyHostToDevice, ix->stream));
      copy(words.p, ids.p, d_src, d_dst, n, nw.p, ni.p);
    }
    B200VS_CUDA(cudaStreamSynchronize(ix->stream));
    words.swap(nw); ids.swap(ni);
  }
  // rows [r0, r0 + n) as packed bytes [n, dim / 8] on the host
  size_t row_bytes() const { return (size_t)ix->dim / 8; }
  void download(int64_t r0, int64_t n, uint8_t* out) const {
    if (n <= 0) return;
    const int nb = ix->dim / 8;
    std::vector<uint32_t> tmp((size_t)n * w);
    B200VS_CUDA(cudaMemcpy(tmp.data(), words.p + (size_t)r0 * w, tmp.size() * 4, cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < n; ++i) memcpy(out + (size_t)i * nb, tmp.data() + (size_t)i * w, nb);
  }
  const void* row_data() const { return words.p; }
  size_t row_pitch() const { return (size_t)w * 4; }  // the packed bytes lead each padded row (little-endian words)
  int64_t bytes() const { return (int64_t)(words.cap * 4 + ids.cap * 8); }
  // the row fields of a tile-scan view; the owner adds the list layout
  TcView view() const {
    TcView v;
    v.vecs = reinterpret_cast<const float*>(words.p); v.ids = ids.p;
    return v;
  }
};

// Shared by both binary types: the float entry points are refused (api.cu), rows arrive packed.
struct BinaryIndex : IndexBase {
  const int nb, w;  // bytes per packed row; 32-bit words per padded row
  BinaryIndex(b200vs_type t, int d, const b200vs_params& p) : IndexBase(t, B200VS_HAMMING, d, p), nb(d / 8), w(words_of(d)) {}

  // packed device rows -> padded words in scratch
  const uint32_t* pad(int64_t n, const uint8_t* x_dev, cudaStream_t s) {
    uint32_t* out = scratch.alloc<uint32_t>((size_t)std::max<int64_t>(n, 1) * w);
    if (n > 0) {
      launch_pad_rows(x_dev, n, nb, out, s);
      launch_count(1);
    }
    return out;
  }
  ScanJob hamming_job(const uint32_t* rows, const long long* ids, long long n) const {
    ScanJob j;
    j.hamming = true;
    j.vecs = reinterpret_cast<const float*>(rows); j.ids = ids; j.d = w; j.mode = 0; j.n = n;
    return j;
  }
  // IndexBinary::range_search takes an int radius (flat.cc:304-308): the float is truncated toward zero, and hits have
  // dis < radius.  Every radius above dim + 1 admits the same rows, so larger values (and +inf) are clamped there first.
  // The threshold of a range search (0 for top-k); a NaN radius is refused before anything is launched.
  float radius_threshold(const SearchReq& r) const {
    if (!r.range) return 0.f;
    if (std::isnan(r.radius)) fail(B200VS_EILLEGAL_PARAMETERS, "radius is NaN");
    return std::trunc(std::min(r.radius, (float)(dim + 1)));
  }
  // the exact scan j of a top-k search (the timed dominant scan), or of a range search with threshold thr
  static void finish_job(const SearchReq& r, float thr, ScanJob& j) {
    if (r.range) { j.has_thr = true; j.thr_raw = thr; }
    else j.dominant = true;
  }

};

// ============================================================================================
// Binary Flat: IndexBinaryFlat under IndexBinaryIDMap2 (vector_index_flat.cc:99-102, :121-264), with the float Flat's
// policies: append, tombstone, compaction at half dead.
// ============================================================================================
struct BinaryFlatIndex : BinaryIndex {
  FlatRowMap<BinRows> rowmap{this};

  BinaryFlatIndex(int d, const b200vs_params& p) : BinaryIndex(B200VS_BINARY_FLAT, d, p) {}

  // AddOrUpsert (flat.cc:121-162): duplicate ids in the batch are refused, existing ids are always removed first
  void add(const AddReq& r) override {
    if (r.ids) check_batch_ids_unique(r.n, r.ids);
    WriteHold hold(this);
    Staged st;
    stage(r, nb, false, st);
    if (!r.ids) check_batch_ids_unique(r.n, st.ids);
    rowmap.add(r.n, pad(r.n, static_cast<const uint8_t*>(st.x), stream), st.ids_dev, st.ids);
  }
  void check_add(const AddReq& r) override { IndexBase::check_add(r); check_batch_ids_unique(r.n, r.ids); }
  // Delete (flat.cc:171-203): ids that are not present are ignored
  int64_t remove(int64_t n, const int64_t* del) override {
    WriteHold hold(this);
    return rowmap.remove(n, del);
  }
  void live_rows(int64_t lo, int64_t hi, RebuildSource& out) override {
    rowmap.live_slots(out.ids, out.slots, lo, hi);
    out.rows = rowmap.store.words.p;
    out.stream = stream;
  }
  // the sources' padded rows in ascending id order in one add
  int64_t rebuild_from(const std::vector<IndexBase*>& srcs, int64_t lo, int64_t hi) override {
    DevBuf<uint32_t> rows;
    DevBuf<long long> ids;
    const int64_t n = sorted_live_rows(this, srcs, lo, hi, w, rows, ids, stream);
    if (n == 0) return 0;
    std::vector<int64_t> h_ids(n);
    B200VS_CUDA(cudaMemcpyAsync(h_ids.data(), ids.p, (size_t)n * 8, cudaMemcpyDeviceToHost, stream));
    B200VS_CUDA(cudaStreamSynchronize(stream));
    rowmap.add(n, rows.p, ids.p, h_ids.data());
    return n;
  }
  ScanJob job(const SearchCtx& sc) const {
    ScanJob j = hamming_job(rowmap.store.words.p, rowmap.store.ids.p, rowmap.rows);
    j.sc = &sc;
    return j;
  }
  // Search / RangeSearch (flat.cc:206-323): Hamming distances are exact, so od is the raw key too
  void search(const SearchReq& r, cudaStream_t s) override {
    refuse_probes(r);
    const float thr = radius_threshold(r);
    const uint32_t* q = pad(r.nq, static_cast<const uint8_t*>(r.xq), s);
    const TcView v = rowmap.view();
    ScanJob j = job(*r.sc);
    if (r.deep) { run_scan_deep(this, j, r.nq, reinterpret_cast<const float*>(q), r.k, r.od, false, r.oi, s); return; }
    if (!r.range && bt_eligible(v, r.nq, r.k, 1, (double)rowmap.rows, *r.sc)) {
      long long* probes = scratch.alloc<long long>(r.nq);
      B200VS_CUDA(cudaMemsetAsync(probes, 0, (size_t)r.nq * 8, s));
      bt_search(this, v, w, r.nq, q, r.k, probes, 1, j, r.od, r.oi, s);
      return;
    }
    finish_job(r, thr, j);
    run_scan(this, j, r.nq, reinterpret_cast<const float*>(q), r.k, r.od, nullptr, r.oi, r.oc, s);
  }
  int64_t count() const override { return rowmap.count(); }
  int64_t deleted_count() const override { return rowmap.ndeleted; }
  int64_t memory_size() const override { return rowmap.store.bytes(); }
  void export_lists(int64_t* list_off, float* vectors, uint8_t* codes, int64_t* out_ids) override {
    if (vectors) fail(B200VS_EILLEGAL_PARAMETERS, "binary indexes export packed rows through codes; vectors must be NULL");
    RwSharedGuard rl(this);
    std::lock_guard<std::mutex> gl(gpu_mu);
    set_device();
    quiesce();
    rowmap.export_rows(list_off, codes, out_ids);
  }
  void pack_lists(int64_t* list_off, void* out_ids, uint8_t* out_rows) override {
    RwSharedGuard rl(this);
    std::lock_guard<std::mutex> gl(gpu_mu);
    set_device();
    quiesce();
    rowmap.pack(list_off, out_ids, out_rows);
  }
};

IndexBase* make_binary_flat(int d, const b200vs_params& p) { return new BinaryFlatIndex(d, p); }

// ============================================================================================
// Binary IVF-Flat: IndexBinaryIVF with an IndexBinaryFlat quantiser (vector_index_ivf_flat.cc:62).  Lists live in the
// IvfLists arena with the float IVF-Flat's relocation and compaction policy; rows move as words.
// ============================================================================================
struct BinaryIvfIndex : BinaryIndex {
  int nlist;  // degenerates to 1 at train time with fewer rows than nlist (ivf_flat.cc:578-641)
  bool trained = false;
  DevBuf<uint32_t> cent;       // [nlist, w] padded binary centroids
  DevBuf<long long> cent_ids;  // iota: the list ids the coarse pass returns
  BinRows store{this};
  IvfLists L;

  BinaryIvfIndex(int d, const b200vs_params& p) : BinaryIndex(B200VS_BINARY_IVF_FLAT, d, p) {
    nlist = p.nlist > 0 ? p.nlist : 2048;  // Constant::kCreateBinaryIvfFlatParamNcentroids (constant.h:180)
  }
  bool is_trained() const override { return trained; }
  int export_nlist() const override { return nlist; }
  int nlist_now() const override { return nlist; }

  // packed centroids [k, dim / 8] (host); the writer hold is taken
  void install_centroids(const uint8_t* host_c, int k) {
    nlist = k;
    scratch.reset(stream);
    uint8_t* raw = scratch.alloc<uint8_t>((size_t)k * nb);
    B200VS_CUDA(cudaMemcpyAsync(raw, host_c, (size_t)k * nb, cudaMemcpyHostToDevice, stream));
    const uint32_t* st = pad(k, raw, stream);
    cent.free(); cent_ids.free();
    cent.reserve((size_t)k * w, 0, stream);
    cent_ids.reserve(k, 0, stream);
    B200VS_CUDA(cudaMemcpyAsync(cent.p, st, (size_t)k * w * 4, cudaMemcpyDeviceToDevice, stream));
    launch_iota(cent_ids.p, k, stream);
    B200VS_CUDA(cudaStreamSynchronize(stream));
    L.init(k, stream);
    store.reset();
    trained = true;
  }

  // trained-state blob: int64 hdr[4] = {magic 'IVFB', nlist, dim, metric}; uint8 centroids[nlist * dim / 8]
  static constexpr int64_t kStateMagic = 0x42465649;
  void state_header(void* blob, int k) const {
    const int64_t hdr[4] = {kStateMagic, k, dim, (int64_t)metric};
    memcpy(blob, hdr, 32);
  }
  void set_state(const void* blob, size_t len) override {
    WriteHold hold(this);
    if (len < 32) fail(B200VS_EILLEGAL_PARAMETERS, "state blob too short");
    const int64_t* hdr = (const int64_t*)blob;
    if (hdr[0] != kStateMagic || hdr[2] != dim || hdr[3] != B200VS_HAMMING) fail(B200VS_EILLEGAL_PARAMETERS, "bad binary IVF state blob");
    if (hdr[1] <= 0 || hdr[1] > (1 << 24)) fail(B200VS_EILLEGAL_PARAMETERS, "bad list count in state blob");
    const int k = (int)hdr[1];
    if (len < 32 + (size_t)k * nb) fail(B200VS_EILLEGAL_PARAMETERS, "state blob truncated");
    install_centroids((const uint8_t*)blob + 32, k);
  }
  int64_t get_state(void* blob, size_t cap) override {
    RwSharedGuard rl(this);
    if (!trained) return 0;
    const size_t need = 32 + (size_t)nlist * nb;
    if (!blob || cap < need) return (int64_t)need;
    set_device();
    state_header(blob, nlist);
    std::vector<uint32_t> tmp((size_t)nlist * w);
    B200VS_CUDA(cudaMemcpyAsync(tmp.data(), cent.p, tmp.size() * 4, cudaMemcpyDeviceToHost, stream));
    B200VS_CUDA(cudaStreamSynchronize(stream));
    for (int c = 0; c < nlist; ++c) memcpy((uint8_t*)blob + 32 + (size_t)c * nb, tmp.data() + (size_t)c * w, nb);
    return (int64_t)need;
  }

  // IndexBinaryIVF::train: binary_to_real (bit i = byte i >> 3, bit i & 7, LSB first -> 2b - 1), faiss::Clustering with L2
  // on the +-1 rows (kmeans_gpu: same subsample permutation, seed, iterations and split_clusters as IVF-Flat), and
  // real_to_binary (bit set where the coordinate is > 0).  Only the training subsample is expanded to floats: the rows
  // kmeans_gpu would draw, in its order, so it sees exactly what it would see on the whole expanded set.
  void train(int64_t n, const void* x) override {
    WriteHold hold(this);
    if (trained) return;  // ivf_flat.cc:670-672
    train_locked(n, static_cast<const uint8_t*>(x), nullptr);
  }
  // train's rule with rw and gpu_mu held, on host packed rows x, or (x_words) on padded rows already on the device,
  // whose sample is expanded to +-1 floats there
  void train_locked(int64_t n, const uint8_t* x, const uint32_t* x_words) {
    const int k = n < nlist ? 1 : nlist;  // "data size too small, nlist degenerate to 1"
    std::vector<uint8_t> bin;
    kmeans_locked(n, x, x_words, k, bin);
    install_centroids(bin.data(), k);
    train_rows = n;
  }
  // train_locked's clustering into k <= n packed centroids bin [k, dim / 8], leaving the index as it is (rw and gpu_mu held)
  void kmeans_locked(int64_t n, const uint8_t* x, const uint32_t* x_words, int k, std::vector<uint8_t>& bin) {
    const int max_pts = 256, niter = 10;
    const int64_t seed = 1234;
    std::vector<int64_t> pick;
    int64_t m = n;
    if (n > (int64_t)k * max_pts) { kmeans_rand_perm(pick, n, seed); m = (int64_t)k * max_pts; }
    // kmeans_gpu holds the +-1 sample on the device: refuse a sample that cannot fit there before it is built on the host
    // (dim 32768 with nlist 2048 is 68 GB); EINTERNAL like any device allocation failure, and the index stays untrained
    size_t free_b = 0, total_b = 0;
    B200VS_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const double sample_b = (double)m * dim * 4;
    if (sample_b > (double)free_b)
      fail(B200VS_EINTERNAL, "binary training sample of " + std::to_string((long long)(sample_b / 1e6)) + " MB (+-1 floats) does not fit in " +
                                 std::to_string((long long)(free_b / 1000000)) + " MB of free device memory");
    DevBuf<long long> iota;
    std::vector<float> c;
    auto assign = [&](const float* xd, int64_t mm, const float* cd, int kk, long long* out) {
      ScanJob j;
      j.vecs = cd; j.ids = iota.p; j.d = dim; j.mode = 0; j.n = kk;
      const int64_t chunk = 32768;
      for (int64_t a = 0; a < mm; a += chunk) {
        const auto mark = scratch.mark();
        run_scan(this, j, std::min(chunk, mm - a), xd + (size_t)a * dim, 1, nullptr, nullptr, out + a, nullptr, stream);
        scratch.release(mark);
      }
    };
    auto prepare_ids = [&](int kk) { iota.reserve(kk, 0, stream); launch_iota(iota.p, kk, stream); };
    // if the device fills up in between, kmeans_gpu's DevBuf::reserve fails the same way (CudaError -> EINTERNAL)
    if (x_words) {
      DevBuf<long long> d_pick;
      DevBuf<float> pm1;
      if (!pick.empty()) {
        d_pick.reserve(m, 0, stream);
        B200VS_CUDA(cudaMemcpyAsync(d_pick.p, pick.data(), (size_t)m * 8, cudaMemcpyHostToDevice, stream));
      }
      pm1.reserve((size_t)m * dim, 0, stream);
      launch_expand_pm1(x_words, d_pick.p, m, w, dim, pm1.p, stream);
      kmeans_gpu_dev(this, dim, m, pm1.p, k, niter, max_pts, seed, c, assign, prepare_ids);
    } else {
      std::vector<float> pm1((size_t)m * dim);  // bad_alloc -> EINTERNAL, index stays untrained
      for (int64_t i = 0; i < m; ++i) {
        const uint8_t* row = x + (size_t)(pick.empty() ? i : pick[i]) * nb;
        float* o = pm1.data() + (size_t)i * dim;
        for (int b = 0; b < dim; ++b) o[b] = ((row[b >> 3] >> (b & 7)) & 1) ? 1.0f : -1.0f;
      }
      kmeans_gpu(this, B200VS_L2, dim, m, pm1.data(), k, niter, max_pts, seed, c, assign, prepare_ids);
    }
    bin.assign((size_t)k * nb, 0);
    for (int ci = 0; ci < k; ++ci)
      for (int b = 0; b < dim; ++b)
        if (c[(size_t)ci * dim + b] > 0.0f) bin[(size_t)ci * nb + (b >> 3)] |= (uint8_t)(1u << (b & 7));
  }

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
    out.rows = store.words.p;
    out.stream = stream;
  }
  // train on the sources' padded rows in ascending id order, then add them in that order
  int64_t rebuild_from(const std::vector<IndexBase*>& srcs, int64_t lo, int64_t hi) override {
    DevBuf<uint32_t> rows;
    DevBuf<long long> ids;
    const int64_t n = sorted_live_rows(this, srcs, lo, hi, w, rows, ids, stream);
    if (n == 0) return 0;
    train_locked(n, nullptr, rows.p);
    scratch.reset(stream);
    std::vector<int64_t> h_ids(n);
    B200VS_CUDA(cudaMemcpyAsync(h_ids.data(), ids.p, (size_t)n * 8, cudaMemcpyDeviceToHost, stream));
    B200VS_CUDA(cudaStreamSynchronize(stream));
    place_locked(n, rows.p, ids.p, h_ids.data());
    return n;
  }

  int resolve_nprobe(const SearchCtx& sc) const {
    const int np = sc.nprobe > 0 ? sc.nprobe : 80;  // Constant::kSearchBinaryIvfFlatParamNprobe (constant.h:181), ivf_flat.cc:207-209
    return std::min(np, nlist);                    // ivf_flat.cc:234
  }
  int resolve_nprobe_api(const SearchCtx& sc) const override { return resolve_nprobe(sc); }
  // IndexBinaryFlat quantiser over centroid rows [c0, c1) (c1 < 0: every row): the nprobe nearest lists by (Hamming
  // distance, list id), as global list ids, with their distances in out_dist when it is set
  long long* coarse_lists(int64_t nq, const uint32_t* q, int nprobe, cudaStream_t s, long long* out = nullptr, int c0 = 0, int c1 = -1,
                          float* out_dist = nullptr) {
    if (c1 < 0) c1 = nlist;
    long long* probes = out ? out : scratch.alloc<long long>((size_t)nq * nprobe);
    run_scan(this, hamming_job(cent.p + (size_t)c0 * w, cent_ids.p + c0, c1 - c0), nq, reinterpret_cast<const float*>(q), nprobe, nullptr,
             out_dist, probes, nullptr, s);
    return probes;
  }
  // packed query rows; the list-sharded search's coarse step on its slice of the batch (prepared has no meaning for bits)
  void coarse(int64_t nq, const void* xq, bool, int nprobe, int c0, int c1, float* out_score, long long* out_lists, cudaStream_t s) override {
    if (!trained) fail(B200VS_EVECTOR_NOT_TRAIN, "not train");
    if (c0 < 0 || c1 > nlist || c0 >= c1 || nprobe <= 0 || nprobe > c1 - c0) fail(B200VS_EILLEGAL_PARAMETERS, "bad centroid range / nprobe");
    coarse_lists(nq, pad(nq, static_cast<const uint8_t*>(xq), s), nprobe, s, out_lists, c0, c1, out_score);
  }
  // nearest list of n padded rows, ties to the smaller list id (the coarse pass with nprobe = 1), in chunks whose select
  // workspace is handed back before the next
  void assign_words(int64_t n, const uint32_t* st, long long* lists, cudaStream_t s) {
    for (int64_t a = 0; a < n; a += 32768) {
      const auto mark = scratch.mark();
      coarse_lists(std::min<int64_t>(32768, n - a), st + (size_t)a * w, 1, s, lists + a);
      scratch.release(mark);
    }
  }
  // packed rows: the assignment the sender of a list-sharded add routes by (a lane must be held)
  void assign_lists_dev(int64_t n, const void* x_dev, long long* out_lists_dev, cudaStream_t s) override {
    if (!trained) fail(B200VS_EVECTOR_NOT_TRAIN, "not train");
    assign_words(n, pad(n, static_cast<const uint8_t*>(x_dev), s), out_lists_dev, s);
  }
  TcView view() const {
    TcView v = store.view();
    v.arena_rows = L.arena_used; v.list_off = L.d_off.p; v.list_len = L.d_len.p;
    v.nlist = nlist; v.total_chunks = L.total_chunks; v.max_chunks_per_list = L.max_chunks_per_list;
    return v;
  }
  ScanJob list_job(const SearchCtx& sc, const long long* probes, int nprobe) const {
    ScanJob j = hamming_job(store.words.p, store.ids.p, 0);
    j.mode = 1; j.probes = probes; j.nprobe = nprobe; j.list_off = L.d_off.p; j.list_len = L.d_len.p; j.sc = &sc;
    j.avg_candidates = nlist > 0 ? (double)L.total_len() * nprobe / nlist : 0;
    return j;
  }

  // untrained -> refused (ivf_flat.cc:111-113); upsert removes the ids first (:115-118); rows go to
  // the caller's lists (the owner of a list-sharded add) or the nearest ones.  The form has no meaning for bits.
  void add(const AddReq& r) override {
    WriteHold hold(this);
    if (!trained) fail(B200VS_EVECTOR_NOT_TRAIN, "not train");
    Staged st;
    stage(r, nb, false, st);
    place_locked(r.n, pad(r.n, static_cast<const uint8_t*>(st.x), stream), st.ids_dev, st.ids, r.lists, r.upsert);
  }
  // padded device rows st and ids st_ids (in_ids: the same on the host) to the tails of their lists: lists_dev, or (null) the
  // nearest ones, as an upsert (IvfLists::place) when upsert; the writer hold is taken
  void place_locked(int64_t n, const uint32_t* st, const long long* st_ids, const int64_t* in_ids, const long long* lists_dev = nullptr,
                    bool upsert = false) {
    std::vector<long long> h_list;
    IvfLists::row_lists(this, n, lists_dev, h_list, [&](long long* out) { assign_words(n, st, out, stream); });
    L.place(n, h_list.data(), in_ids, st, st_ids, store, upsert);
  }
  // Delete (ivf_flat.cc:162-189): untrained -> OK; nothing removed -> EVECTOR_INVALID (api.cu)
  int64_t remove(int64_t n, const int64_t* del) override {
    WriteHold hold(this);
    if (!trained) return -1;
    return L.remove(n, del, store);
  }

  // Search / RangeSearch (ivf_flat.cc:203-350): untrained -> empty results (:224-227); the range scan is the exact one
  // (:342-345).  A caller's probe table (a list-sharded search) takes the place of the coarse pass.
  void search(const SearchReq& r, cudaStream_t s) override {
    if (!trained) { fill_empty(r, s); return; }
    const SearchCtx& sc = *r.sc;
    const float thr = radius_threshold(r);
    const uint32_t* q = pad(r.nq, static_cast<const uint8_t*>(r.xq), s);
    const int nprobe = r.probes ? r.nprobe : resolve_nprobe(sc);
    const long long* probes = r.probes ? r.probes : coarse_lists(r.nq, q, nprobe, s);
    if (profiling && !r.range) profile_probed(this, probes, r.nq * nprobe, nlist, L.d_len.p, s);
    const TcView v = view();
    ScanJob j = list_job(sc, probes, nprobe);
    if (r.deep) { run_scan_deep(this, j, r.nq, reinterpret_cast<const float*>(q), r.k, r.od, false, r.oi, s); return; }
    if (!r.range && L.live > 0 && bt_eligible(v, r.nq, r.k, nprobe, j.avg_candidates, sc)) {
      bt_search(this, v, w, r.nq, q, r.k, probes, nprobe, j, r.od, r.oi, s);
      return;
    }
    finish_job(r, thr, j);
    run_scan(this, j, r.nq, reinterpret_cast<const float*>(q), r.k, r.od, nullptr, r.oi, r.oc, s);
  }

  int64_t count() const override { return L.live; }
  int64_t deleted_count() const override { return L.dead; }
  int64_t memory_size() const override { return store.bytes() + (int64_t)cent.cap * 4; }
  void export_lists(int64_t* list_off, float* vectors, uint8_t* codes, int64_t* out_ids) override {
    if (vectors) fail(B200VS_EILLEGAL_PARAMETERS, "binary indexes export packed rows through codes; vectors must be NULL");
    RwSharedGuard rl(this);
    std::lock_guard<std::mutex> gl(gpu_mu);
    set_device();
    quiesce();
    L.export_lists(nlist, list_off, store, codes, out_ids);
  }
  void pack_lists(int64_t* list_off, void* out_ids, uint8_t* out_rows) override {
    RwSharedGuard rl(this);
    std::lock_guard<std::mutex> gl(gpu_mu);
    set_device();
    quiesce();
    L.pack(nlist, list_off, store, out_ids, out_rows);
  }
};

IndexBase* make_binary_ivf(int d, const b200vs_params& p) { return new BinaryIvfIndex(d, p); }

static BinaryIvfIndex* as_binary_ivf(IndexBase* ix) {
  auto* p = dynamic_cast<BinaryIvfIndex*>(ix);
  if (!p) fail(B200VS_EINTERNAL, "not a BINARY_IVF_FLAT index");
  return p;
}

void binary_ivf_train_coarse(IndexBase* ix, int64_t n, const uint8_t* x, const uint32_t* x_words, int k, std::vector<uint8_t>& cent) {
  BinaryIvfIndex* b = as_binary_ivf(ix);
  WriteHold hold(b);
  b->kmeans_locked(n, x, x_words, k, cent);
}

void binary_ivf_train_state(IndexBase* ix, const std::vector<uint8_t>& cent, std::vector<unsigned char>& blob) {
  const BinaryIvfIndex* b = as_binary_ivf(ix);
  blob.resize(32 + cent.size());
  b->state_header(blob.data(), (int)(cent.size() / b->nb));
  memcpy(blob.data() + 32, cent.data(), cent.size());
}

}  // namespace b200vs
