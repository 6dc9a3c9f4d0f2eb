// ivf_common.h — row bookkeeping of every index with a row store (Flat, IVF-Flat, IVF-PQ and their binary forms) and the
// GPU k-means shared by the IVF types.
//
// A row store holds an index's device rows: FP32 rows (RowStore, index.cu), padded binary words (BinRows, binary.cu) or PQ
// code rows (CodeRows, ivf_pq.cu), each with a device id per row (-1 = tombstone / unused slot).  The stores share one
// shape, used here as a template argument: grow(cap, keep), reset(), move(src, dst, n), write(rows, ids, slots),
// gather(src, dst, cap), download(r0, n, out) in the export's host format of row_bytes() each, bytes(), the device rows
// row_data() of row_pitch() bytes each (the export format is each row's first row_bytes()), and the members ix (the owning
// index, whose stream and scratch they use) and ids.  The store moves rows; the bookkeeping below decides
// capacities, slots, tombstones, compaction and export order.
//
// Inverted lists live in ONE device arena (rows of the payload array), list l owning rows
// [off, off+len) with capacity cap >= len.  Appends go in place; a full list is relocated to the arena
// tail with 1.5x capacity; deletes and upserts tombstone the rows they replace (id = -1), and a write that tombstoned
// rows ends with a compaction pass that rebuilds the arena when garbage + tombstones outweigh live rows.  Plain appends
// never compact.  Lists stay contiguous so the scan kernels stream them with
// 128-B coalesced loads / TMA tiles.  Replaces faiss::ArrayInvertedLists behind IndexIVFFlat/IndexIVFPQ
// (constructed at src/vector/vector_index_ivf_flat.cc:809-816, vector_index_raw_ivf_pq.cc:554-564).
#pragma once
#include <algorithm>
#include <cmath>
#include <random>
#include <unordered_map>
#include <vector>

#include "index.h"
#include "tc_scan.cuh"

namespace b200vs {

// The snapshot pack (b200vs_save_stage, snapshot.cu): row slots[i] of the device rows `rows` (pitch bytes apart) and its id
// ids[slots[i]] become row i of out_rows (the first row_bytes of it) and out_ids[i], on the host.  One gather kernel packs
// them on the owner's stream, then one device-to-host copy per buffer and one synchronise.
void pack_rows(IndexBase* ix, const std::vector<long long>& slots, const void* rows, size_t pitch, const long long* ids, size_t row_bytes,
               void* out_ids, uint8_t* out_rows);

// ids[r] = -1 for every listed row, on the owner's stream
inline void tombstone_ids(IndexBase* ix, long long* ids, const std::vector<int64_t>& rows) {
  if (rows.empty()) return;
  long long* d_rows = ix->scratch.alloc<long long>(rows.size());
  B200VS_CUDA(cudaMemcpyAsync(d_rows, rows.data(), rows.size() * 8, cudaMemcpyHostToDevice, ix->stream));
  launch_set_ids(ids, d_rows, (int64_t)rows.size(), -1, ix->stream);
  B200VS_CUDA(cudaStreamSynchronize(ix->stream));
}

// The rows of a Flat index (float or binary): appended in order, tombstoned on delete, compacted at half dead.  The one
// "list" of rows [0, rows) is what the tile scan sees.
template <class Store>
struct FlatRowMap {
  Store store;
  int64_t rows = 0;
  std::vector<int64_t> h_ids;
  std::unordered_map<int64_t, int64_t> id2row;
  int64_t ndeleted = 0;
  DevBuf<long long> d_off1;  // the single "list" of a Flat index, for the tile-scan view
  DevBuf<int> d_len1;

  template <class... A>
  explicit FlatRowMap(IndexBase* ix, A... store_args) : store(ix, store_args...) {
    d_off1.reserve(1, 0, ix->stream); d_len1.reserve(1, 0, ix->stream);
    B200VS_CUDA(cudaMemsetAsync(d_off1.p, 0, 8, ix->stream));
    B200VS_CUDA(cudaMemsetAsync(d_len1.p, 0, 4, ix->stream));
    B200VS_CUDA(cudaStreamSynchronize(ix->stream));
  }
  int64_t count() const { return rows - ndeleted; }
  void publish_len() {
    const int len = (int)std::min<int64_t>(rows, 0x7fffffff);
    B200VS_CUDA(cudaMemcpyAsync(d_len1.p, &len, 4, cudaMemcpyHostToDevice, store.ix->stream));
    B200VS_CUDA(cudaStreamSynchronize(store.ix->stream));
  }
  TcView view() const {
    TcView v = store.view();
    set_flat_layout(v, rows, d_off1.p, d_len1.p);
    return v;
  }

  // the rows holding these ids become tombstones (unknown ids are ignored); returns how many
  int64_t tombstone(int64_t n, const int64_t* del) {
    std::vector<int64_t> dead;
    for (int64_t i = 0; i < n; ++i) {
      auto it = id2row.find(del[i]);
      if (it != id2row.end()) { dead.push_back(it->second); id2row.erase(it); }
    }
    tombstone_ids(store.ix, store.ids.p, dead);
    for (int64_t r : dead) h_ids[r] = -1;
    ndeleted += (int64_t)dead.size();
    return (int64_t)dead.size();
  }
  int64_t remove(int64_t n, const int64_t* del) {
    const int64_t r = tombstone(n, del);
    compact_if_needed();
    return r;
  }
  void compact_if_needed() {
    if (ndeleted == 0 || ndeleted * 2 < rows) return;
    std::vector<long long> src, dst;
    src.reserve(rows - ndeleted);
    for (int64_t r = 0; r < rows; ++r) if (h_ids[r] >= 0) src.push_back(r);
    const int64_t live = (int64_t)src.size();
    dst.resize(live);
    for (int64_t i = 0; i < live; ++i) dst[i] = i;
    store.gather(src, dst, std::max<int64_t>(1024, live * 5 / 4));
    std::vector<int64_t> nh(live);
    id2row.clear();
    for (int64_t i = 0; i < live; ++i) { nh[i] = h_ids[src[i]]; id2row[nh[i]] = i; }
    h_ids.swap(nh);
    rows = live; ndeleted = 0;
    publish_len();
  }
  // VectorIndexFlat::AddOrUpsert, vector_index_flat.cc:121-162: rows holding one of the ids are removed first, then the n
  // device rows x / ids_dev (ids_host: the same ids on the host, unique) are appended in order
  template <class Row>
  void add(int64_t n, const Row* x, const long long* ids_dev, const int64_t* ids_host) {
    tombstone(n, ids_host);
    const int64_t cap = (int64_t)store.ids.cap;
    if (rows + n > cap) store.grow(std::max<int64_t>(rows + n, std::max<int64_t>(1024, cap * 3 / 2)), rows);
    std::vector<long long> slots(n);
    for (int64_t i = 0; i < n; ++i) slots[i] = rows + i;
    store.write(x, ids_dev, slots);
    B200VS_CUDA(cudaStreamSynchronize(store.ix->stream));
    h_ids.resize(rows + n);
    for (int64_t i = 0; i < n; ++i) { h_ids[rows + i] = ids_host[i]; id2row[ids_host[i]] = rows + i; }
    rows += n;
    publish_len();
    compact_if_needed();
  }
  // the live (id, row) pairs with lo <= id <= hi in row order
  void live_slots(std::vector<int64_t>& out_ids, std::vector<long long>& out_rows, int64_t lo = 0, int64_t hi = INT64_MAX) const {
    for (int64_t r = 0; r < rows; ++r)
      if (h_ids[r] >= 0 && h_ids[r] >= lo && h_ids[r] <= hi) { out_ids.push_back(h_ids[r]); out_rows.push_back(r); }
  }
  // export_rows' output through the device pack
  void pack(int64_t* list_off, void* out_ids, uint8_t* out_rows) const {
    std::vector<int64_t> ids;
    std::vector<long long> slots;
    live_slots(ids, slots);
    if ((int64_t)slots.size() != count()) fail(B200VS_EINTERNAL, "row bookkeeping out of step with the live count");
    list_off[0] = 0; list_off[1] = (int64_t)slots.size();
    pack_rows(store.ix, slots, store.row_data(), store.row_pitch(), store.ids.p, store.row_bytes(), out_ids, out_rows);
  }
  // drop every row, keep the buffers
  void clear() {
    rows = 0; ndeleted = 0;
    h_ids.clear(); id2row.clear();
    publish_len();
  }
  // the live rows in row order: out (rows in the store's host format, nullable) and out_ids (nullable).  Without
  // tombstones the rows are downloaded straight into out, so a large export holds no second host copy.
  void export_rows(int64_t* list_off, uint8_t* out, int64_t* out_ids) const {
    if (list_off) { list_off[0] = 0; list_off[1] = count(); }
    const size_t rb = store.row_bytes();
    std::vector<uint8_t> all;
    if (out && ndeleted) all.resize((size_t)rows * rb);
    if (out) store.download(0, rows, ndeleted ? all.data() : out);
    int64_t o = 0;
    for (int64_t r = 0; r < rows; ++r) {
      if (h_ids[r] < 0) continue;
      if (out_ids) out_ids[o] = h_ids[r];
      if (out && ndeleted) memcpy(out + (size_t)o * rb, all.data() + (size_t)r * rb, rb);
      ++o;
    }
  }
};

struct ListMeta {
  int64_t off = 0;
  int32_t len = 0;  // rows in use (live + tombstones)
  int32_t cap = 0;
  int32_t dead = 0;
};

struct IvfLists {
  std::vector<ListMeta> lists;
  std::vector<int64_t> h_ids;  // arena mirror of ids (-1 = tombstone / unused)
  std::unordered_multimap<int64_t, uint64_t> where;  // id -> (list << 32 | pos)
  int64_t arena_used = 0, arena_cap = 0;
  int64_t live = 0, dead = 0, garbage = 0;
  int64_t total_chunks = 0;      // sum of ceil(len / 512) — tensor-core work-item bound (tc_scan.cuh TC_CHUNK = 512)
  int max_chunks_per_list = 0;
  DevBuf<long long> d_off;
  DevBuf<int> d_len;

  void init(int nlist, cudaStream_t s) {
    lists.assign(nlist, ListMeta());
    h_ids.clear(); where.clear();
    arena_used = arena_cap = 0;
    live = dead = garbage = 0;
    d_off.free(); d_len.free();
    d_off.reserve(nlist, 0, s);
    d_len.reserve(nlist, 0, s);
    upload(s);
  }
  int64_t total_len() const { return live + dead; }

  void upload(cudaStream_t s) {
    const size_t n = lists.size();
    std::vector<long long> off(n);
    std::vector<int> len(n);
    total_chunks = 0; max_chunks_per_list = 0;
    for (size_t i = 0; i < n; ++i) {
      off[i] = lists[i].off; len[i] = lists[i].len;
      const int c = (lists[i].len + 511) / 512;
      total_chunks += c; max_chunks_per_list = std::max(max_chunks_per_list, c);
    }
    B200VS_CUDA(cudaMemcpyAsync(d_off.p, off.data(), n * 8, cudaMemcpyHostToDevice, s));
    B200VS_CUDA(cudaMemcpyAsync(d_len.p, len.data(), n * 4, cudaMemcpyHostToDevice, s));
    B200VS_CUDA(cudaStreamSynchronize(s));  // host vectors die here
  }

  static int32_t round32(int64_t v) { return (int32_t)((v + 31) / 32 * 32); }

  void check_lists(int64_t n, const long long* h_list) const {
    for (int64_t i = 0; i < n; ++i)
      if (h_list[i] < 0 || h_list[i] >= (long long)lists.size()) fail(B200VS_EILLEGAL_PARAMETERS, "list id out of range");
  }

  // n rows go to the tails of their lists h_list: device rows x and ids ids_dev, the same ids on the host in h_ids_in.  A
  // list without room is relocated to the arena tail with 1.5x capacity, and the arena grows by 1.5x when that runs out.
  // upsert: every row already holding one of the ids is tombstoned first, and the write ends as a delete does.
  template <class Store, class Row>
  void place(int64_t n, const long long* h_list, const int64_t* h_ids_in, const Row* x, const long long* ids_dev, Store& store,
             bool upsert = false) {
    check_lists(n, h_list);
    const int64_t replaced = upsert ? tombstone(n, h_ids_in, store) : 0;
    std::vector<int> need(lists.size(), 0);
    for (int64_t i = 0; i < n; ++i) need[h_list[i]]++;
    struct Rel { int64_t src, dst; int32_t len; };
    std::vector<Rel> rels;
    const int64_t used_before = arena_used;
    for (size_t l = 0; l < lists.size(); ++l) {
      if (need[l] == 0) continue;
      ListMeta& m = lists[l];
      if (m.len + need[l] <= m.cap) continue;
      const int32_t ncap = round32(std::max<int64_t>(64, ((int64_t)m.len + need[l]) * 3 / 2));
      rels.push_back({m.off, arena_used, m.len});
      garbage += m.cap;
      m.off = arena_used; m.cap = ncap;
      arena_used += ncap;
    }
    if (arena_used > arena_cap) {
      const int64_t ncap = std::max<int64_t>(arena_used, arena_cap * 3 / 2);
      store.grow(ncap, used_before);
      arena_cap = ncap;
    }
    h_ids.resize(arena_cap, -1);
    for (const Rel& r : rels) {
      if (r.len == 0) continue;
      store.move(r.src, r.dst, (int64_t)r.len);
      std::copy(h_ids.begin() + r.src, h_ids.begin() + r.src + r.len, h_ids.begin() + r.dst);
    }
    std::vector<long long> slots(n);
    for (int64_t i = 0; i < n; ++i) {
      const int l = (int)h_list[i];
      ListMeta& m = lists[l];
      slots[i] = m.off + m.len;
      where.emplace(h_ids_in[i], ((uint64_t)l << 32) | (uint32_t)m.len);
      h_ids[slots[i]] = h_ids_in[i];
      m.len++;
    }
    live += n;
    store.write(x, ids_dev, slots);
    upload(store.ix->stream);
    if (replaced) compact_if_needed(store);
  }

  // the inverted list of each of n rows an add places, on the device (returned) and in h_list: the caller's device lists,
  // or (lists null) those assign(out) writes, the nearest; on the owner's stream
  template <class Assign>
  static const long long* row_lists(IndexBase* ix, int64_t n, const long long* lists, std::vector<long long>& h_list, Assign assign) {
    if (!lists) {
      long long* out = ix->scratch.alloc<long long>(n);
      assign(out);
      lists = out;
    }
    h_list.resize(n);
    B200VS_CUDA(cudaMemcpyAsync(h_list.data(), lists, (size_t)n * 8, cudaMemcpyDeviceToHost, ix->stream));
    B200VS_CUDA(cudaStreamSynchronize(ix->stream));
    return lists;
  }

  // faiss remove_ids(IDSelectorBatch): every row whose id matches becomes a tombstone; returns how many
  template <class Store>
  int64_t tombstone(int64_t n, const int64_t* del, Store& store) {
    std::vector<int64_t> rows;
    for (int64_t i = 0; i < n; ++i) {
      auto range = where.equal_range(del[i]);
      for (auto it = range.first; it != range.second; ++it) {
        const int l = (int)(it->second >> 32);
        const uint32_t pos = (uint32_t)(it->second & 0xffffffffu);
        const int64_t row = lists[l].off + pos;
        if (h_ids[row] < 0) continue;
        h_ids[row] = -1;
        lists[l].dead++;
        rows.push_back(row);
        live--; dead++;
      }
      where.erase(range.first, range.second);
    }
    tombstone_ids(store.ix, store.ids.p, rows);
    return (int64_t)rows.size();
  }
  // a delete: the rows holding these ids become tombstones, then the arena is compacted if needed; returns how many
  template <class Store>
  int64_t remove(int64_t n, const int64_t* del, Store& store) {
    const int64_t r = tombstone(n, del, store);
    compact_if_needed(store);
    return r;
  }

  // The end of every write that tombstones rows (remove, an upsert's place): when garbage and tombstones outweigh the live
  // rows, a fresh arena, list by list in list order, each list holding its live rows in order with room for 1/4 more + 32.
  // Plain appends do not come here: under them relocation garbage alone outgrows the live rows, and a compaction would
  // only re-allocate the arena the appends are about to grow again.
  template <class Store>
  void compact_if_needed(Store& store) {
    if (garbage + dead <= std::max<int64_t>(live, 4096)) return;
    std::vector<ListMeta> nl(lists.size());
    std::vector<long long> src, dst;
    int64_t used = 0;
    for (size_t l = 0; l < lists.size(); ++l) {
      const ListMeta& m = lists[l];
      const int32_t nlive = m.len - m.dead;
      ListMeta& pm = nl[l];
      pm.off = used;
      pm.cap = nlive ? round32((int64_t)nlive * 5 / 4 + 32) : 0;
      for (int p = 0; p < m.len; ++p) {
        if (h_ids[m.off + p] < 0) continue;
        src.push_back(m.off + p);
        dst.push_back(pm.off + pm.len);
        pm.len++;
      }
      used += pm.cap;
    }
    std::vector<int64_t> nids(std::max<int64_t>(used, 1), -1);
    for (size_t i = 0; i < src.size(); ++i) nids[dst[i]] = h_ids[src[i]];
    store.gather(src, dst, std::max<int64_t>(used, 1));
    lists.swap(nl);
    h_ids.swap(nids);
    arena_used = used;
    arena_cap = std::max<int64_t>(used, 1);
    garbage = 0; dead = 0;
    where.clear();
    for (size_t l = 0; l < lists.size(); ++l)
      for (int p = 0; p < lists[l].len; ++p) where.emplace(h_ids[lists[l].off + p], ((uint64_t)l << 32) | (uint32_t)p);
    upload(store.ix->stream);
  }

  // b200vs_reserve_lists on an empty index: one arena allocation holding every list at its final size (+ 1/16 slack), and a
  // tail for lists that still outgrow their reservation, so bulk builds never relocate a list or re-allocate the arena.
  // Every size is checked before anything changes.
  template <class Store>
  void reserve(const int64_t* rows_per_list, int n_lists, Store& store) {
    if (n_lists != (int)lists.size()) fail(B200VS_EILLEGAL_PARAMETERS, "reserve_lists: list count does not match the trained index");
    if (live + dead > 0) fail(B200VS_EILLEGAL_PARAMETERS, "reserve_lists needs an empty index");
    for (int l = 0; l < n_lists; ++l)
      if (rows_per_list[l] < 0 || rows_per_list[l] >= (1LL << 31) - 64) fail(B200VS_EILLEGAL_PARAMETERS, "reserve_lists: bad list size");
    int64_t used = 0;
    for (int l = 0; l < n_lists; ++l) {
      const int64_t want = rows_per_list[l];
      ListMeta& m = lists[l];
      m.off = used; m.len = 0; m.dead = 0;
      m.cap = want ? round32(want + want / 16 + 32) : 0;
      used += m.cap;
    }
    arena_used = used;
    arena_cap = used + std::max<int64_t>(used / 64, 4096);
    store.reset();
    store.grow(arena_cap, 0);
    B200VS_CUDA(cudaMemsetAsync(store.ids.p, 0xFF, (size_t)arena_cap * 8, store.ix->stream));  // id -1 = unused slot
    h_ids.assign(arena_cap, -1);
    upload(store.ix->stream);
  }

  // the live rows of list l in list order: the first `cap` of them go to out (the store's host format, nullable) and
  // out_ids (nullable); returns how many there are.  An untrained index has no lists yet, so none.
  template <class Store>
  int64_t export_list(int l, int64_t cap, const Store& store, uint8_t* out, int64_t* out_ids) const {
    if (l >= (int)lists.size()) return 0;
    const ListMeta& m = lists[l];
    const size_t rb = store.row_bytes();
    std::vector<uint8_t> buf;
    if (out && m.len) { buf.resize((size_t)m.len * rb); store.download(m.off, m.len, buf.data()); }
    int64_t o = 0;
    for (int p = 0; p < m.len; ++p) {
      const int64_t id = h_ids[m.off + p];
      if (id < 0) continue;
      if (o < cap) {
        if (out_ids) out_ids[o] = id;
        if (out) memcpy(out + (size_t)o * rb, buf.data() + (size_t)p * rb, rb);
      }
      ++o;
    }
    return o;
  }
  // the live (id, arena row) pairs with lo <= id <= hi, list after list in list order, as export_lists gives them
  void live_slots(std::vector<int64_t>& out_ids, std::vector<long long>& out_rows, int64_t lo = 0, int64_t hi = INT64_MAX) const {
    for (const ListMeta& m : lists)
      for (int p = 0; p < m.len; ++p) {
        const int64_t id = h_ids[m.off + p];
        if (id >= 0 && id >= lo && id <= hi) { out_ids.push_back(id); out_rows.push_back(m.off + p); }
      }
  }
  // export_lists' output through the device pack
  template <class Store>
  void pack(int nlist, int64_t* list_off, const Store& store, void* out_ids, uint8_t* out_rows) const {
    std::vector<long long> slots;
    slots.reserve((size_t)live);
    for (int l = 0; l < nlist; ++l) {
      list_off[l] = (int64_t)slots.size();
      if (l >= (int)lists.size()) continue;
      const ListMeta& m = lists[l];
      for (int p = 0; p < m.len; ++p)
        if (h_ids[m.off + p] >= 0) slots.push_back(m.off + p);
    }
    list_off[nlist] = (int64_t)slots.size();
    if ((int64_t)slots.size() != live) fail(B200VS_EINTERNAL, "list bookkeeping out of step with the live count");
    pack_rows(store.ix, slots, store.row_data(), store.row_pitch(), store.ids.p, store.row_bytes(), out_ids, out_rows);
  }
  // every list's live rows, list after list; list_off[nlist + 1] (nullable) gets where each list starts
  template <class Store>
  void export_lists(int nlist, int64_t* list_off, const Store& store, uint8_t* out, int64_t* out_ids) const {
    int64_t o = 0;
    for (int l = 0; l < nlist; ++l) {
      if (list_off) list_off[l] = o;
      o += export_list(l, INT64_MAX, store, out ? out + (size_t)o * store.row_bytes() : nullptr, out_ids ? out_ids + o : nullptr);
    }
    if (list_off) list_off[nlist] = o;
  }
};

// Per-centroid sums of the assigned rows in 64-bit fixed point (row value * scale, rounded): integer addition does not
// depend on the order in which rows arrive, so training gives the same centroids on every run.
void launch_kmeans_accumulate(const float* x, const long long* assign, int64_t n, int d, double scale, long long* sums,
                              int* counts, cudaStream_t s);

// the first rows of this permutation of [0, m) are k-means' training subsample (seed) and initial centroids (seed + 1)
inline void kmeans_rand_perm(std::vector<int64_t>& perm, int64_t m, int64_t sd) {
  perm.resize(m);
  for (int64_t i = 0; i < m; ++i) perm[i] = i;
  std::mt19937 mt((unsigned)sd);
  for (int64_t i = 0; i + 1 < m; ++i) { int64_t i2 = i + (int64_t)(mt() % (unsigned long)(m - i)); std::swap(perm[i], perm[i2]); }
}

// The Lloyd iterations of kmeans_gpu / kmeans_gpu_dev on the m prepared sample rows xd (device); init_src is the same rows
// on the host (initial centroids, fixed-point scale).
template <class AssignFn, class PrepFn>
void kmeans_lloyd(IndexBase* ix, int d, int64_t m, const float* xd, const float* init_src, int k, int niter, int64_t seed,
                  std::vector<float>& cent, AssignFn assign, PrepFn prepare_ids) {
  cudaStream_t s = ix->stream;
  DevBuf<float> cd;
  DevBuf<long long> sums;
  DevBuf<int> counts;
  DevBuf<long long> asg;
  cent.assign((size_t)k * d, 0.f);
  if (m == k) { memcpy(cent.data(), init_src, (size_t)m * d * 4); return; }
  {
    std::vector<int64_t> perm;
    kmeans_rand_perm(perm, m, seed + 1);
    for (int i = 0; i < k; ++i) memcpy(&cent[(size_t)i * d], init_src + (size_t)perm[i] * d, (size_t)d * 4);
  }
  // fixed-point scale: a sum of m rows of magnitude <= amax stays below 2^62
  float amax = 0.f;
  for (size_t i = 0; i < (size_t)m * d; ++i) amax = std::max(amax, std::fabs(init_src[i]));
  const double scale = amax > 0.f && std::isfinite(amax) ? std::ldexp(1.0, 62 - std::ilogb((double)amax * (double)m) - 1) : 1.0;
  prepare_ids(k);
  cd.reserve((size_t)k * d, 0, s);
  sums.reserve((size_t)k * d, 0, s);
  counts.reserve(k, 0, s);
  asg.reserve(m, 0, s);
  std::vector<long long> hs((size_t)k * d);
  std::vector<int> hc(k);
  for (int it = 0; it < niter; ++it) {
    B200VS_CUDA(cudaMemcpyAsync(cd.p, cent.data(), (size_t)k * d * 4, cudaMemcpyHostToDevice, s));
    assign(xd, m, cd.p, k, asg.p);
    B200VS_CUDA(cudaMemsetAsync(sums.p, 0, (size_t)k * d * 8, s));
    B200VS_CUDA(cudaMemsetAsync(counts.p, 0, (size_t)k * 4, s));
    launch_kmeans_accumulate(xd, asg.p, m, d, scale, sums.p, counts.p, s);
    B200VS_CUDA(cudaMemcpyAsync(hs.data(), sums.p, (size_t)k * d * 8, cudaMemcpyDeviceToHost, s));
    B200VS_CUDA(cudaMemcpyAsync(hc.data(), counts.p, (size_t)k * 4, cudaMemcpyDeviceToHost, s));
    B200VS_CUDA(cudaStreamSynchronize(s));
    std::vector<float> hassign(k);
    for (int c = 0; c < k; ++c) {
      hassign[c] = (float)hc[c];
      if (hc[c] == 0) continue;
      const float inv = 1.0f / (float)hc[c];
      for (int j = 0; j < d; ++j) cent[(size_t)c * d + j] = (float)((double)hs[(size_t)c * d + j] / scale) * inv;
    }
    // split_clusters (faiss public algorithm): refill empty clusters from big ones with a +-1/1024 perturbation
    const float EPS = 1 / 1024.;
    std::mt19937 mt(1234);
    for (int ci = 0; ci < k; ++ci) {
      if (hassign[ci] != 0) continue;
      int cj;
      for (cj = 0;; cj = (cj + 1) % k) {
        const float p = (hassign[cj] - 1.0f) / (float)(m - k);
        const float r = mt() / float(mt.max());
        if (r < p) break;
      }
      memcpy(&cent[(size_t)ci * d], &cent[(size_t)cj * d], (size_t)d * 4);
      for (int j = 0; j < d; ++j) {
        if (j % 2 == 0) { cent[(size_t)ci * d + j] *= 1 + EPS; cent[(size_t)cj * d + j] *= 1 - EPS; }
        else            { cent[(size_t)ci * d + j] *= 1 - EPS; cent[(size_t)cj * d + j] *= 1 + EPS; }
      }
      hassign[ci] = hassign[cj] / 2;
      hassign[cj] -= hassign[ci];
    }
  }
  ix->launch_count(2 * niter);
}

// faiss::Clustering-shaped Lloyd k-means with the assignment step on the GPU (public algorithm; the
// reference reaches it through index_->train at vector_index_ivf_flat.cc:695 / raw_ivf_pq.cc:485).
// x_host RAW rows; cosine rows are normalised on the device first.  `assign(xd, m, cd, k, out)` labels m device
// rows against the k device centroids cd; `prepare_ids(k)` lets the caller size its centroid-id array.
template <class AssignFn, class PrepFn>
void kmeans_gpu(IndexBase* ix, b200vs_metric metric, int d, int64_t n, const float* x_host, int k, int niter,
                int max_pts, int64_t seed, std::vector<float>& cent, AssignFn assign, PrepFn prepare_ids) {
  cudaStream_t s = ix->stream;
  std::vector<float> sub;
  const float* xs = x_host;
  int64_t m = n;
  if (n > (int64_t)k * max_pts) {
    std::vector<int64_t> perm;
    kmeans_rand_perm(perm, n, seed);
    m = (int64_t)k * max_pts;
    sub.resize((size_t)m * d);
    for (int64_t i = 0; i < m; ++i) memcpy(&sub[(size_t)i * d], x_host + (size_t)perm[i] * d, (size_t)d * 4);
    xs = sub.data();
  }
  DevBuf<float> xd;
  xd.reserve((size_t)m * d, 0, s);
  B200VS_CUDA(cudaMemcpyAsync(xd.p, xs, (size_t)m * d * 4, cudaMemcpyHostToDevice, s));
  if (metric == B200VS_COSINE) launch_normalize_faiss(xd.p, m, d, s);
  B200VS_CUDA(cudaStreamSynchronize(s));
  std::vector<float> hx;  // normalised copy for initialisation when cosine
  const float* init_src = xs;
  if (metric == B200VS_COSINE) {
    hx.resize((size_t)m * d);
    B200VS_CUDA(cudaMemcpy(hx.data(), xd.p, (size_t)m * d * 4, cudaMemcpyDeviceToHost));
    init_src = hx.data();
  }
  kmeans_lloyd(ix, d, m, xd.p, init_src, k, niter, seed, cent, assign, prepare_ids);
}

// gather_rows: dst row i = src row (rows ? rows[i] : i), `words` 32-bit words per row, on s
void launch_gather_words(const uint32_t* src, const long long* rows, int64_t n, int words, uint32_t* dst, cudaStream_t s);

// The subsample kmeans_gpu draws (the first k * max_pts rows of kmeans_rand_perm(n, seed), or every row), as indices of the
// n rows, uploaded to `out` on s; returns its size m and leaves out empty when every row is used.
int64_t kmeans_sample_rows(IndexBase* ix, int64_t n, int k, int max_pts, int64_t seed, DevBuf<long long>& out);

// kmeans_gpu on n rows that are already on the device and already prepared (cosine rows normalised: they are not
// normalised again): the same subsample, drawn by kmeans_rand_perm and gathered on the device, the same initial
// centroids, iterations and split_clusters, so the centroids equal kmeans_gpu's on the same rows.
template <class AssignFn, class PrepFn>
void kmeans_gpu_dev(IndexBase* ix, int d, int64_t n, const float* x_dev, int k, int niter, int max_pts, int64_t seed,
                    std::vector<float>& cent, AssignFn assign, PrepFn prepare_ids) {
  cudaStream_t s = ix->stream;
  DevBuf<long long> pick;
  const int64_t m = kmeans_sample_rows(ix, n, k, max_pts, seed, pick);
  DevBuf<float> xd;
  const float* xs = x_dev;
  if (pick.p) {
    xd.reserve((size_t)m * d, 0, s);
    launch_gather_words(reinterpret_cast<const uint32_t*>(x_dev), pick.p, m, d, reinterpret_cast<uint32_t*>(xd.p), s);
    xs = xd.p;
  }
  std::vector<float> hx((size_t)m * d);
  B200VS_CUDA(cudaMemcpyAsync(hx.data(), xs, (size_t)m * d * 4, cudaMemcpyDeviceToHost, s));
  B200VS_CUDA(cudaStreamSynchronize(s));
  kmeans_lloyd(ix, d, m, xs, hx.data(), k, niter, seed, cent, assign, prepare_ids);
}

// The rows of a rebuild in ascending id order, on the sources' device (b200vs_rebuild_from[_range],
// b200vs_shard_rebuild_from): the live rows with lo <= id <= hi of every source (IndexBase::live_rows, filtered on the host
// before anything is uploaded), concatenated in source order, sorted by id with one stable device radix sort whose values
// encode (source, slot), so rows that share an id keep source order and then each source's storage order, and gathered by
// one kernel from each source's row store (`words` 32-bit words per row) into out_rows.  An id held by more than one source
// is refused with EVECTOR_ID_DUPLICATED (the gather compares adjacent sorted ids).  ix counts the launches.  Runs on stream s
// and returns the row count with s synchronised.
int64_t sorted_live_rows(IndexBase* ix, const std::vector<IndexBase*>& srcs, int64_t lo, int64_t hi, int words, DevBuf<uint32_t>& out_rows,
                         DevBuf<long long>& out_ids, cudaStream_t s);
// One block of device rows for the sort below: n rows of `words` words at rows, their ids at ids, both on the device.
struct DeviceRows {
  int64_t n;
  const long long* ids;
  const uint32_t* rows;
};
// the same sort and gather of every row of up to kRebuildMaxSources device row blocks, concatenated in block order (one
// block: no duplicate check); an id held by two blocks is refused with EVECTOR_ID_DUPLICATED
void sorted_live_rows(IndexBase* ix, const std::vector<DeviceRows>& blocks, int words, DevBuf<uint32_t>& out_rows, DevBuf<long long>& out_ids,
                      cudaStream_t s);
// b200vs_rebuild_from[_range] and the row-sharded shard rebuilds: fill dst from the live rows with lo <= id <= hi of srcs
// (distinct, dst not among them) under the sources' reader locks and dst's writer hold, taken in address order.  flat_ok:
// FLAT and BINARY_FLAT are served.
int64_t rebuild_range(IndexBase* dst, const std::vector<IndexBase*>& srcs, int64_t lo, int64_t hi, bool flat_ok);
// out [m, dim] = the +-1 floats (binary_to_real: bit set -> 1, else -1) of padded binary rows words [.., w] (rows ? rows[i] : i)
void launch_expand_pm1(const uint32_t* words, const long long* rows, int64_t m, int w, int dim, float* out, cudaStream_t s);
// the refusals b200vs_rebuild_from[_range] shares for every type and source: dst must be empty, untrained, another index of
// the same type, metric, dimension, result-deciding creation parameters and device
void check_rebuild_pair(const IndexBase& dst, const IndexBase& src);

void check_batch_ids_unique(int64_t n, const int64_t* ids);

// The stable device radix sort of n (id, value) pairs by id (ids are >= 0), the rebuild's and the brute-force range
// search's: keys_out / vals_out get the n pairs in ascending id order, pairs with equal ids in their input order.  temp(bytes)
// hands out the sort's temporary storage.  On stream s.
void sort_by_id(int64_t n, const long long* keys, long long* keys_out, const long long* vals, long long* vals_out,
                const std::function<void*(size_t)>& temp, cudaStream_t s);

}  // namespace b200vs
