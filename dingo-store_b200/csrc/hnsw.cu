// hnsw.cu — HNSW index: graph built on the host, searched on the GPU (per-hop candidate-distance batches).
//
// Replaces hnswlib::HierarchicalNSW<float> behind VectorIndexHnsw (src/vector/vector_index_hnsw.cc:135-184 ctor:
// L2Space / InnerProductSpace, cosine = NormalizeVectorForHnsw + IP; M = nlinks, efConstruction, seed 100;
// :203-254 Upsert -> addPoint; :318-485 Search -> searchKnn(q, k, filter), sticky setEf :426-428, result popped
// back-to-front so it is ascending :400-419, distance emitted as hnswlib returns it :374 (L2: squared L2; IP
// space: 1 - ip); RangeSearch -> EVECTOR_NOT_SUPPORT :487-493).
//
// Graph construction follows the published hnswlib 0.7 algorithm (the fork dingodb/hnswlib@1964db3e is not
// vendored): level = (int)(-ln(U) / ln(M)) with std::default_random_engine(seed); maxM0 = 2M; search with
// ef_construction; heuristic neighbour selection; bidirectional links with heuristic shrink.  It runs on the host
// (single writer, deterministic) with the hooked AVX-512 distance order, so a graph built here equals the graph
// the CPU path builds from the same insertion order; the device holds a mirror that is refreshed lazily.
//
// The host graph, the device mirror and the state blob share one layout (DESIGN §5): level-0 lists in link0, the upper-level
// lists of node i in one linkup pool from up_off[i].  hnsw_links addresses a list on both sides; parse_state reads a blob.
//
// Search (hnsw_search_kernel) and batched construction (hnsw_build_search_kernel) share one device graph walk: one
// 128-thread CTA per query or row; greedy descent through the upper levels, then the reference's searchBaseLayerST at one
// level, whose hops score the <= 32 unvisited neighbours of a node together (32 quads, exact AVX-512 order, so the
// traversal is the CPU traversal).  See "The walk of one CTA" below and DESIGN §4.4.
#include <algorithm>
#include <cmath>
#include <queue>
#include <memory>
#include <mutex>
#include <random>
#include <thread>
#include <unordered_set>

#include <cub/cub.cuh>

#include "index.h"
#include "scan_kernels.cuh"
#include "tc_scan.cuh"

namespace b200vs {

namespace {

// ---------------- host distance: same evaluation order as src/simd/distances_avx512.cc:48-143 ----------------
template <bool L2>
float host_avx512_order(const float* x, const float* y, size_t d) {
  float acc[16];
  for (int l = 0; l < 16; ++l) acc[l] = 0.0f;
  while (d >= 16) {
    for (int l = 0; l < 16; ++l) {
      if (L2) { const float t = x[l] - y[l]; acc[l] = acc[l] + t * t; }
      else    { acc[l] = acc[l] + x[l] * y[l]; }
    }
    x += 16; y += 16; d -= 16;
  }
  float m1[8], m2[4];
  for (int l = 0; l < 8; ++l) m1[l] = acc[8 + l] + acc[l];
  if (d >= 8) {
    for (int l = 0; l < 8; ++l) { if (L2) { const float t = x[l] - y[l]; m1[l] = m1[l] + t * t; } else m1[l] = m1[l] + x[l] * y[l]; }
    x += 8; y += 8; d -= 8;
  }
  for (int l = 0; l < 4; ++l) m2[l] = m1[4 + l] + m1[l];
  if (d >= 4) {
    for (int l = 0; l < 4; ++l) { if (L2) { const float t = x[l] - y[l]; m2[l] = m2[l] + t * t; } else m2[l] = m2[l] + x[l] * y[l]; }
    x += 4; y += 4; d -= 4;
  }
  if (d > 0) {
    float bx[4] = {0, 0, 0, 0}, by[4] = {0, 0, 0, 0};
    for (size_t i = 0; i < d; ++i) { bx[i] = x[i]; by[i] = y[i]; }
    for (int l = 0; l < 4; ++l) { if (L2) { const float t = bx[l] - by[l]; m2[l] = m2[l] + t * t; } else m2[l] = m2[l] + bx[l] * by[l]; }
  }
  return (m2[0] + m2[1]) + (m2[2] + m2[3]);
}

typedef uint32_t tableint;
typedef std::pair<float, tableint> HPair;
struct ByFirst { bool operator()(HPair const& a, HPair const& b) const noexcept { return a.first < b.first; } };
typedef std::priority_queue<HPair, std::vector<HPair>, ByFirst> HHeap;

// [count, links...] of a node at a level, in the layout of the host graph, the device mirror and the state blob
__host__ __device__ __forceinline__ unsigned int* hnsw_links(unsigned int* link0, const int64_t* up_off, unsigned int* linkup, int maxM,
                                                             int maxM0, unsigned int node, int level) {
  return level == 0 ? link0 + (size_t)node * (maxM0 + 1) : linkup + up_off[node] + (size_t)(level - 1) * (maxM + 1);
}

struct HostGraph {
  int metric, d;
  size_t M, maxM, maxM0, efc;
  double mult;
  std::default_random_engine rng;
  int64_t n = 0;  // nodes inserted; during an add, the per-node arrays also hold the call's laid-out slots beyond n
  int maxlevel = -1;
  tableint enterpoint = (tableint)-1;
  std::vector<float> data;
  std::vector<int64_t> labels;
  std::vector<int> levels;
  std::vector<tableint> link0;
  std::vector<int64_t> up_off{0};  // node i's upper-level lists: linkup[up_off[i], up_off[i + 1]), levels[i] · (maxM + 1) entries
  std::vector<tableint> linkup;
  std::vector<uint8_t> deleted;
  std::unordered_map<int64_t, tableint> lookup;
  std::vector<uint32_t> visited;
  uint32_t tag = 0;
  int64_t ndeleted = 0;
  // concurrent insertion (hnswlib's locking scheme): one lock per node for its link lists, one for the entry point /
  // max level, one for slot allocation + label map; every worker owns a visited-tag array
  struct VisitCtx { std::vector<uint32_t> visited; uint32_t tag = 0; };
  std::unique_ptr<std::mutex[]> node_mu;
  int64_t node_mu_cap = 0;
  struct Locks { std::mutex global_mu, alloc_mu; };
  std::unique_ptr<Locks> lk{new Locks()};  // (heap-held so that the graph object stays movable)

  void init(int metric_, int d_, int M_, int efc_, int64_t seed) {
    metric = metric_; d = d_; M = M_; maxM = M_; maxM0 = 2 * (size_t)M_; efc = std::max((size_t)efc_, (size_t)M_);
    mult = 1 / log(1.0 * M_);
    rng.seed((unsigned)seed);
  }
  void reserve_locks(int64_t ncap) {
    if (ncap <= node_mu_cap) return;
    node_mu.reset(new std::mutex[(size_t)ncap]);
    node_mu_cap = ncap;
  }
  std::vector<int> draw_levels(int64_t k, std::default_random_engine& r) const {  // the next k nodes' levels, in node order
    std::uniform_real_distribution<double> U(0.0, 1.0);
    std::vector<int> lev((size_t)k);
    for (int& l : lev) l = (int)(-log(U(r)) * mult);
    return lev;
  }
  void extend_up_off(std::vector<int64_t>& off, const std::vector<int>& lev) const {  // pool offsets of nodes with levels lev
    for (int l : lev) off.push_back(off.back() + (int64_t)l * (int64_t)(maxM + 1));
  }
  // Lays out the slots of a call's nodes, with levels lev, after the slots laid out so far: levels, pool offsets, zeroed
  // level-0 blocks and pool slots, and room for their rows.  Nothing grows while add_point (or the batched commit) fills them.
  void append_nodes(const std::vector<int>& lev) {
    const size_t n1 = levels.size() + lev.size();
    levels.insert(levels.end(), lev.begin(), lev.end());
    extend_up_off(up_off, lev);
    link0.resize(n1 * (maxM0 + 1), 0);
    linkup.resize((size_t)up_off.back(), 0);
    data.resize(n1 * d); labels.resize(n1); deleted.resize(n1, 0); visited.resize(n1, 0);
  }
  void take_label(int64_t label, tableint c) {  // node c takes the label; the label's old node, if live, becomes a tombstone
    auto it = lookup.find(label);
    if (it != lookup.end() && !deleted[it->second]) { deleted[it->second] = 1; ++ndeleted; }
    lookup[label] = c;
  }
  const float* vec(tableint i) const { return &data[(size_t)i * d]; }
  float dist(const float* a, const float* b) const {
    if (metric == B200VS_L2) return host_avx512_order<true>(a, b, d);
    return 1.0f - host_avx512_order<false>(a, b, d);
  }
  tableint* ll(tableint i, int level) { return hnsw_links(link0.data(), up_off.data(), linkup.data(), (int)maxM, (int)maxM0, i, level); }

  template <bool MT>
  HHeap search_layer(tableint ep, const float* q, int layer, VisitCtx* vc = nullptr) {
    std::vector<uint32_t>& visited = MT ? vc->visited : this->visited;
    uint32_t& tag = MT ? vc->tag : this->tag;
    if (++tag == 0) { std::fill(visited.begin(), visited.end(), 0u); tag = 1; }
    HHeap top, cand;
    float lower;
    if (!deleted[ep]) { const float d0 = dist(q, vec(ep)); top.emplace(d0, ep); lower = d0; cand.emplace(-d0, ep); }
    else { lower = std::numeric_limits<float>::max(); cand.emplace(-lower, ep); }
    visited[ep] = tag;
    while (!cand.empty()) {
      HPair cur = cand.top();
      if ((-cur.first) > lower && top.size() == efc) break;
      cand.pop();
      std::unique_lock<std::mutex> nl;
      if (MT) nl = std::unique_lock<std::mutex>(node_mu[cur.second]);
      const tableint* l = ll(cur.second, layer);
      const size_t size = l[0];
      for (size_t j = 1; j <= size; ++j) {
        const tableint c = l[j];
        if (visited[c] == tag) continue;
        visited[c] = tag;
        const float d1 = dist(q, vec(c));
        if (top.size() < efc || lower > d1) {
          cand.emplace(-d1, c);
          if (!deleted[c]) top.emplace(d1, c);
          if (top.size() > efc) top.pop();
          if (!top.empty()) lower = top.top().first;
        }
      }
    }
    return top;
  }
  void heuristic(HHeap& top, size_t lim) {
    if (top.size() < lim) return;
    HHeap closest;
    std::vector<HPair> ret;
    while (!top.empty()) { closest.emplace(-top.top().first, top.top().second); top.pop(); }
    while (!closest.empty()) {
      if (ret.size() >= lim) break;
      const HPair cur = closest.top();
      const float dq = -cur.first;
      closest.pop();
      bool good = true;
      for (const HPair& s : ret) if (dist(vec(s.second), vec(cur.second)) < dq) { good = false; break; }
      if (good) ret.push_back(cur);
    }
    for (const HPair& p : ret) top.emplace(-p.first, p.second);
  }
  template <bool MT>
  tableint connect(tableint cur_c, HHeap& top, int level) {
    const size_t mcur = level ? maxM : maxM0;
    heuristic(top, M);
    std::vector<tableint> sel;
    while (!top.empty()) { sel.push_back(top.top().second); top.pop(); }
    const tableint next_ep = sel.back();
    tableint* l = ll(cur_c, level);
    l[0] = (tableint)sel.size();
    for (size_t i = 0; i < sel.size(); ++i) l[1 + i] = sel[i];
    for (size_t idx = 0; idx < sel.size(); ++idx) {
      std::unique_lock<std::mutex> nl;
      if (MT) nl = std::unique_lock<std::mutex>(node_mu[sel[idx]]);
      tableint* lo = ll(sel[idx], level);
      const size_t sz = lo[0];
      if (sz < mcur) { lo[1 + sz] = cur_c; lo[0] = (tableint)(sz + 1); }
      else {
        HHeap cands;
        cands.emplace(dist(vec(cur_c), vec(sel[idx])), cur_c);
        for (size_t j = 0; j < sz; ++j) cands.emplace(dist(vec(lo[1 + j]), vec(sel[idx])), lo[1 + j]);
        heuristic(cands, mcur);
        int k = 0;
        while (!cands.empty()) { lo[1 + k] = cands.top().second; cands.pop(); ++k; }
        lo[0] = (tableint)k;
      }
    }
    return next_ep;
  }
  // addPoint for a NEW label (replacing an existing label = mark the old node deleted, then insert).  MT = several threads
  // insert at once (the reference's ParallelFor over addPoint, vector_index_hnsw.cc:229-243).  The caller has laid out the
  // node's slot (append_nodes, which drew its level) and reserved the locks, so no container grows while workers run.
  template <bool MT>
  void add_point(const float* x, int64_t label, VisitCtx* vc = nullptr) {
    tableint cur_c;
    {
      std::unique_lock<std::mutex> al;
      if (MT) al = std::unique_lock<std::mutex>(lk->alloc_mu);
      cur_c = (tableint)n++;
      take_label(label, cur_c);
    }
    const int curlevel = levels[cur_c];
    std::unique_lock<std::mutex> own;
    if (MT) own = std::unique_lock<std::mutex>(node_mu[cur_c]);
    std::unique_lock<std::mutex> gl;
    if (MT) gl = std::unique_lock<std::mutex>(lk->global_mu);
    const int maxlevelcopy = maxlevel;
    if (MT && curlevel <= maxlevelcopy) gl.unlock();
    tableint cur = enterpoint;
    memcpy(&data[(size_t)cur_c * d], x, sizeof(float) * d);
    labels[cur_c] = label;
    const float* q = vec(cur_c);
    if ((int)cur != -1) {
      if (curlevel < maxlevelcopy) {
        float curdist = dist(q, vec(cur));
        for (int level = maxlevelcopy; level > curlevel; --level) {
          bool changed = true;
          while (changed) {
            changed = false;
            std::unique_lock<std::mutex> nl;
            if (MT) nl = std::unique_lock<std::mutex>(node_mu[cur]);
            const tableint* l = ll(cur, level);
            const int size = l[0];
            for (int i = 1; i <= size; ++i) {
              const float dd = dist(q, vec(l[i]));
              if (dd < curdist) { curdist = dd; cur = l[i]; changed = true; }
            }
          }
        }
      }
      for (int level = std::min(curlevel, maxlevelcopy); level >= 0; --level) {
        HHeap top = search_layer<MT>(cur, q, level, vc);
        cur = connect<MT>(cur_c, top, level);
      }
    } else { enterpoint = 0; maxlevel = curlevel; }
    if (curlevel > maxlevelcopy) { enterpoint = cur_c; maxlevel = curlevel; }
  }
};

// The one reader of a state blob (layout and refusals: DESIGN §5): a fresh graph with the parameters of `like`.  A blob whose
// graph the host builder or the device walk could not traverse within its arrays is refused.
HostGraph parse_state(const HostGraph& like, const void* blob, size_t len) {
  HostGraph H;
  H.init(like.metric, like.d, (int)like.M, (int)like.efc, 100);
  auto refuse = [](const char* why) { fail(B200VS_EILLEGAL_PARAMETERS, std::string("bad HNSW state blob (") + why + ")"); };
  auto pad8 = [](uint64_t v) { return (v + 7) / 8 * 8; };
  const char* base = (const char*)blob;
  int64_t hdr[8], pool;
  if (len < 64) refuse("truncated");
  memcpy(hdr, base, 64);
  if (hdr[0] != 0x57534E48 || hdr[2] != H.d || hdr[3] != (int64_t)H.M || hdr[4] != (int64_t)H.maxM0) refuse("header");
  const int64_t n = hdr[1];
  if (n < 0 || n > (1LL << 31)) refuse("row count");
  const uint64_t o_off = pad8(64 + (uint64_t)n * 4), o_link0 = o_off + (uint64_t)(n + 1) * 8;
  if (len < o_link0) refuse("truncated");
  memcpy(&pool, base + o_off + (uint64_t)n * 8, 8);
  if (pool < 0 || pool > (int64_t)(len / 4)) refuse("link pool");
  const uint64_t n0 = (uint64_t)n * (H.maxM0 + 1), o_pool = o_link0 + n0 * 4, o_data = pad8(o_pool + (uint64_t)pool * 4);
  const uint64_t o_labels = pad8(o_data + (uint64_t)n * H.d * 4), o_end = o_labels + (uint64_t)n * 8;
  if (len < o_end) refuse("truncated");
  auto take = [&](auto& v, uint64_t off, uint64_t count) { v.resize(count); if (count) memcpy(v.data(), base + off, count * sizeof(v[0])); };
  take(H.levels, 64, n); take(H.up_off, o_off, n + 1); take(H.link0, o_link0, n0); take(H.linkup, o_pool, pool);
  take(H.data, o_data, (uint64_t)n * H.d); take(H.labels, o_labels, n);
  H.deleted.assign(n, 0);
  if (len >= o_end + n) take(H.deleted, o_end, n);  // the optional trailing tombstones
  H.visited.assign(n, 0);
  if (n == 0 && (hdr[5] != -1 || hdr[6] != (int64_t)(tableint)-1)) refuse("empty graph with an entry point");
  if (n > 0 && (hdr[6] < 0 || hdr[6] >= n || H.levels[hdr[6]] != hdr[5])) refuse("entry point");
  H.n = n; H.maxlevel = (int)hdr[5]; H.enterpoint = (tableint)hdr[6];
  if (H.up_off[0] != 0) refuse("pool offsets");
  for (int64_t i = 0; i < n; ++i) {  // node i's level and pool slots (up_off[i] <= pool: the sum cannot overflow), then its lists
    if (H.levels[i] < 0 || H.levels[i] > H.maxlevel) refuse("level");
    if (H.up_off[i + 1] != H.up_off[i] + (int64_t)H.levels[i] * (int64_t)(H.maxM + 1) || H.up_off[i + 1] > pool) refuse("pool offsets");
    for (int l = 0; l <= H.levels[i]; ++l) {
      const tableint* ls = H.ll((tableint)i, l);
      if (ls[0] > (l ? H.maxM : H.maxM0)) refuse("list count");
      for (tableint j = 1; j <= ls[0]; ++j)
        if (ls[j] >= (uint64_t)n || H.levels[ls[j]] < l) refuse("link target");
    }
    if (H.deleted[i] > 1) refuse("tombstone");
    H.ndeleted += H.deleted[i];
    if (!H.deleted[i]) H.lookup[H.labels[i]] = (tableint)i;
  }
  return H;
}

// ---------------- device graph walk: search and batched construction ----------------
// The device mirror of HostGraph's first n nodes.  The construction's link and reverse kernels write its link lists.
struct HnswDev {
  const float* data;
  const long long* labels;
  unsigned int* link0;
  const int64_t* up_off;
  unsigned int* linkup;
  const unsigned char* deleted;
  long long n;
  int d, maxM, maxM0, maxlevel, efc;
  unsigned int enterpoint;
  int has_deletions, M;
  __device__ __forceinline__ unsigned int* links(unsigned int node, int level) const { return hnsw_links(link0, up_off, linkup, maxM, maxM0, node, level); }
};

// HostGraph::dist on the device: quad lane t's part of the exact AVX-512 order, then hnswlib's InnerProductDistance
// (1 - ip) for IP and cosine
template <bool L2>
__device__ __forceinline__ float hnsw_distance(const float* x, const float* y, int d, int t, bool vec) {
  const float v = quad_distance<L2>(x, y, d, t, vec);
  return L2 ? v : __fsub_rn(1.0f, v);
}

constexpr int HNSW_THREADS = 128;   // one CTA per query: warp 0 walks the graph, all 32 quads score a hop's neighbours together
constexpr int HNSW_CAND_SMEM = 1024; // candidate-heap entries kept in shared memory (the levels near the root); deeper ones spill to global
// Heap form: the visited set admits every node to the candidate heap at most once, so n + 1 entries per query always
// suffice.  When nq · (n + 1) entries exceed this budget the queries run in chunks of fewer CTAs.
constexpr size_t HNSW_CAND_POOL_BYTES = 512ull << 20;
constexpr size_t HNSW_SMEM_LIMIT = 200 * 1024;  // dynamic shared memory of every HNSW kernel

struct HeapEnt { float d; unsigned int id; };

// Dynamic shared memory of a walk kernel: the query (padded to 16 bytes), the result array or heap [ef + 1], then the
// candidate heap's shared part [HNSW_CAND_SMEM], which the merged-array form uses as its second array.
__host__ __device__ __forceinline__ size_t walk_qbytes(int d) { return ((size_t)d * 4 + 15) / 16 * 16; }
size_t walk_smem_bytes(int d, int ef) { return walk_qbytes(d) + (size_t)(ef + 1) * sizeof(HeapEnt) + (size_t)HNSW_CAND_SMEM * sizeof(HeapEnt); }

// Binary heap operated by ONE lane.  MAXH: largest distance on top.  Entries [0, nsm) live in shared memory, the rest in
// global memory: a sift walks a root-to-leaf path, whose upper levels (the hot ones) are the shared part.
struct HeapRef {
  HeapEnt* sm;
  HeapEnt* gl;
  int nsm;
  __device__ __forceinline__ HeapEnt get(int i) const { return i < nsm ? sm[i] : gl[i]; }
  __device__ __forceinline__ void set(int i, HeapEnt e) const { if (i < nsm) sm[i] = e; else gl[i] = e; }
};
template <bool MAXH>
__device__ __forceinline__ bool h_before(float a, float b) { return MAXH ? a > b : a < b; }
template <bool MAXH>
__device__ void h_push(const HeapRef& h, int& n, float d, unsigned int id) {
  int i = n++;
  while (i > 0) {
    const int p = (i - 1) >> 1;
    const HeapEnt pe = h.get(p);
    if (h_before<MAXH>(d, pe.d)) { h.set(i, pe); i = p; } else break;
  }
  HeapEnt e; e.d = d; e.id = id;
  h.set(i, e);
}
template <bool MAXH>
__device__ void h_pop(const HeapRef& h, int& n) {
  const HeapEnt last = h.get(--n);
  int i = 0;
  for (;;) {
    int c = 2 * i + 1;
    if (c >= n) break;
    HeapEnt ce = h.get(c);
    if (c + 1 < n) { const HeapEnt c2 = h.get(c + 1); if (h_before<MAXH>(c2.d, ce.d)) { ce = c2; ++c; } }
    if (h_before<MAXH>(ce.d, last.d)) { h.set(i, ce); i = c; } else break;
  }
  if (n > 0) h.set(i, last);
}

// The walk of one CTA (128 threads), shared by the search and the construction search.  Warp 0 runs hnswlib's control flow:
// greedy descent of the upper levels, then a base walk at one level, which takes the next node to expand, reads its link
// list 32 neighbours at a time and keeps the unvisited ones in list order; then ALL 32 quads of the CTA compute those rows'
// distances in one round (exact AVX-512 order, so the traversal is the CPU traversal).  Two block barriers per batch of
// <= 32 neighbours.  The base walk has two forms, which differ in how they pick the next node and take in a scored batch:
// - merged array (FAST: no id filter, no tombstones, so every accepted neighbour enters both of hnswlib's queues): the two
//   binary heaps collapse into ONE ascending array T of the best <= ef nodes with an "expanded" flag per entry.  The next
//   node is the first unexpanded entry of T; a batch is merged into T by all 128 threads at once (each thread places one
//   old entry and at most one new one at its rank), instead of ~30 sift-up / sift-down sequences executed by a single lane
//   at one dependent instruction per ~25 ns — that lone-lane heap work was 80 % of a hop.
// - two heaps (searchBaseLayerST): lane 0 pops the closest candidate and applies the heap updates in neighbour order; the
//   candidate heap spills to global memory past HNSW_CAND_SMEM entries.
// The visited set, the order in which nodes are expanded and the result are those of searchBaseLayerST in both forms
// (exact-distance ties between different nodes, which std::priority_queue orders by heap position, are the one place the
// merged array can differ).
struct Cursor {  // warp 0: the node being expanded and how far into its link list the walk is
  unsigned int node;
  int size, c0;
  bool expanding;
};

template <bool L2>
struct Walk {
  const HnswDev& g;
  const float* qs;    // the query, in shared memory
  unsigned int* vis;  // the visited bitset
  float* s_d;         // [32] in shared memory: the distances of a scoring round
  unsigned int* s_id; // [32] in shared memory: the nodes of a scoring round
  int* s_m;           // in shared memory: rows to score this round; -1 = the walk is over
  // g.d; this thread's quad and lane in it.  The two kernels spell the quad index (and the candidate heap's address) in
  // different but equal ways: ptxas allocates registers differently for each spelling, and these are the ones that keep every
  // instantiation of both kernels within its register allocation and free of new spills (DESIGN §4.4).
  int d, quad, t;
  bool vec;           // rows are 16-byte aligned

  // distances of s_id[0, m) -> s_d[0, m): one row per quad, every thread of the CTA calls (m <= 32)
  __device__ __forceinline__ void score(int m) const {
    const float v = hnsw_distance<L2>(g.data + (size_t)s_id[quad < m ? quad : 0] * d, qs, d, t, vec);
    if (quad < m && t == 0) s_d[quad] = v;
  }
  __device__ __forceinline__ float score_one(unsigned int node) const {
    if (threadIdx.x == 0) s_id[0] = node;
    __syncthreads();
    score(1);
    __syncthreads();
    return s_d[0];
  }
  // Warp 0: the next <= 32 unvisited neighbours at `level` of the node being expanded, marked visited and packed in list
  // order into s_id.  When the node's list is used up, next(node) picks the node to expand next, or returns false when the
  // walk is over.  Returns the batch size, -1 when the walk is over.
  template <class Next>
  __device__ __forceinline__ int collect(Cursor& c, int level, Next& next) const {
    const int lane = threadIdx.x & 31;
    for (;;) {
      if (!c.expanding) {
        if (!next(c.node)) return -1;
        c.size = (int)g.links(c.node, level)[0];
        c.c0 = 0;
        c.expanding = true;
      }
      if (c.c0 >= c.size) { c.expanding = false; continue; }
      const unsigned int* l = g.links(c.node, level) + 1 + c.c0;
      const int cnt = min(32, c.size - c.c0);
      c.c0 += 32;
      unsigned int nb = 0;
      bool fresh = false;
      if (lane < cnt) { nb = l[lane]; fresh = ((vis[nb >> 5] >> (nb & 31)) & 1u) == 0u; }
      const unsigned int mask = __ballot_sync(0xffffffffu, fresh);
      if (fresh) {
        atomicOr(&vis[nb >> 5], 1u << (nb & 31));
        s_id[__popc(mask & ((1u << lane) - 1u))] = nb;
      }
      const int m = __popc(mask);
      if (m > 0) return m;
    }
  }
  // One round of a base walk: warp 0 collects the next batch, the CTA scores it into s_d.  Returns its size (-1: the walk is
  // over), the same on every thread.
  template <class Next>
  __device__ __forceinline__ int round(Cursor& c, int level, Next& next) const {
    __syncthreads();  // (A) the walk's arrays complete, s_d / s_id of the previous round consumed
    if ((threadIdx.x >> 5) == 0) {
      const int m = collect(c, level, next);
      if ((threadIdx.x & 31) == 0) *s_m = m;
    }
    __syncthreads();  // (B) s_id / s_m published
    const int m = *s_m;
    if (m >= 0) {
      score(m);
      __syncthreads();  // (C) s_d complete
    }
    return m;
  }
};

// Greedy descent through the levels from_level down to stop_level + 1, moving from (cur, curdist) to any closer neighbour
// until none is closer.  Every thread tracks the same state.
template <bool L2>
__device__ __forceinline__ void descend(const Walk<L2>& w, int from_level, int stop_level, unsigned int& cur, float& curdist) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int level = from_level; level > stop_level; --level) {
    bool changed = true;
    while (changed) {
      changed = false;
      __builtin_assume(level > 0);  // an upper level: links() needs no level-0 branch
      const unsigned int* l = w.g.links(cur, level);
      const int size = (int)l[0];
      for (int c0 = 0; c0 < size; c0 += 32) {
        const int m = min(32, size - c0);
        __syncthreads();  // previous round's s_d / s_id fully consumed
        if (warp == 0 && lane < m) w.s_id[lane] = l[1 + c0 + lane];
        __syncthreads();
        w.score(m);
        __syncthreads();
        for (int i = 0; i < m; ++i) {
          const float dd = w.s_d[i];
          if (dd < curdist) { curdist = dd; cur = w.s_id[i]; changed = true; }
        }
      }
    }
  }
}

// a before b in the merged walk's order: the float order, with every NaN after every number (and NaNs equal)
__device__ __forceinline__ bool d_before(float a, float b) { return a < b || (b != b && a == a); }

// Base walk at `level`, merged-array form, from (cur, curdist) with capacity ef.  T (id bit 31 = expanded) and T2 are the
// two buffers of the merge, [ef] each; on return T holds the ascending result and the return value is its length.
template <bool L2>
__device__ __forceinline__ int walk_merged(const Walk<L2>& w, int level, int ef, unsigned int cur, float curdist, HeapEnt*& T, HeapEnt* T2) {
  const int lane = threadIdx.x & 31;
  int ntop = 1;
  if (threadIdx.x == 0) { T[0].d = curdist; T[0].id = cur; w.vis[cur >> 5] |= 1u << (cur & 31); }
  auto next = [&](unsigned int& node) {  // first unexpanded entry = closest open candidate
    int idx = -1;
    for (int b0 = 0; b0 < ntop && idx < 0; b0 += 32) {
      const int i = b0 + lane;
      const bool open = i < ntop && (T[i].id >> 31) == 0u;
      const unsigned msk = __ballot_sync(0xffffffffu, open);
      if (msk) idx = b0 + __ffs(msk) - 1;
    }
    if (idx < 0) return false;
    node = T[idx].id;
    __syncwarp();
    if (lane == 0) T[idx].id = node | 0x80000000u;
    return true;
  };
  Cursor c{};
  for (;;) {
    const int m = w.round(c, level, next);
    if (m < 0) break;
    // merge the m scored neighbours into T (ascending, old entries first among equals), keep the best ef.  The ranks are
    // counted in an order that puts NaN (an inner product that overflowed to +inf and -inf) after every number, so the
    // destinations always form a permutation.  With plain float compares a NaN broke that: two entries took one slot,
    // another slot of T2 kept stale shared memory, and its id was walked.
    for (int tix = threadIdx.x; tix < ntop; tix += HNSW_THREADS) {
      const HeapEnt e = T[tix];
      int cnt = 0;
      for (int j = 0; j < m; ++j) cnt += d_before(w.s_d[j], e.d) ? 1 : 0;
      if (tix + cnt < ef) T2[tix + cnt] = e;
    }
    if (threadIdx.x < m) {
      const float dj = w.s_d[threadIdx.x];
      int rank = 0;
      for (int i = 0; i < m; ++i) rank += (d_before(w.s_d[i], dj) || (!d_before(dj, w.s_d[i]) && i < (int)threadIdx.x)) ? 1 : 0;
      int lo = 0, hi = ntop;  // number of old entries not after dj
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (!d_before(dj, T[mid].d)) lo = mid + 1; else hi = mid; }
      if (rank + lo < ef) { HeapEnt e; e.d = dj; e.id = w.s_id[threadIdx.x]; T2[rank + lo] = e; }
    }
    ntop = min(ef, ntop + m);
    HeapEnt* tmp = T; T = T2; T2 = tmp;
  }
  __syncthreads();
  return ntop;
}

// Base walk at `level`, two-heap form, from (cur, curdist) with capacity ef: top = the result max-heap [ef + 1], cand = the
// candidate min-heap.  allowed(node): the node may enter the result (else it is only traversed).  strict_stop: the walk
// stops at a candidate farther than the result only once the result holds ef nodes.  Returns the size of top on thread 0.
template <bool L2, class Allowed>
__device__ __forceinline__ int walk_heaps(const Walk<L2>& w, int level, int ef, bool strict_stop, Allowed allowed, unsigned int cur,
                                          float curdist, const HeapRef& top, const HeapRef& cand) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int ntop = 0, ncand = 0;
  float lower = 3.402823466e+38f;
  if (warp == 0) {
    const bool ok = allowed(cur);
    if (lane == 0) {
      if (ok) { h_push<true>(top, ntop, curdist, cur); h_push<false>(cand, ncand, curdist, cur); }
      else h_push<false>(cand, ncand, 3.402823466e+38f, cur);
      w.vis[cur >> 5] |= 1u << (cur & 31);
    }
    lower = ok ? curdist : 3.402823466e+38f;
  }
  auto next = [&](unsigned int& node) {  // pop the closest candidate unless the walk stops here
    int go = 0;
    if (lane == 0 && ncand > 0) {
      const HeapEnt ce = cand.get(0);
      const bool stop = ce.d > lower && (ntop == ef || !strict_stop);
      if (!stop) { node = ce.id; h_pop<false>(cand, ncand); go = 1; }
    }
    go = __shfl_sync(0xffffffffu, go, 0);
    if (!go) return false;
    node = __shfl_sync(0xffffffffu, node, 0);
    return true;
  };
  Cursor c{};
  for (;;) {
    const int m = w.round(c, level, next);
    if (m < 0) break;
    if (warp == 0) {
      const unsigned int amask = __ballot_sync(0xffffffffu, lane < m && allowed(w.s_id[lane]));
      if (lane == 0) {
        for (int i = 0; i < m; ++i) {
          const float dd = w.s_d[i];
          if (ntop < ef || lower > dd) {
            h_push<false>(cand, ncand, dd, w.s_id[i]);  // fresh nodes only: ncand <= n < the pool's n + 1 entries
            if ((amask >> i) & 1u) h_push<true>(top, ntop, dd, w.s_id[i]);
            if (ntop > ef) h_pop<true>(top, ntop);
            if (ntop > 0) lower = top.get(0).d;
          }
        }
      }
      lower = __shfl_sync(0xffffffffu, lower, 0);
    }
  }
  return ntop;
}

// Search: one CTA per query.  Descent to level 0 from the entry point, then the base walk with ef: the merged-array form
// when FAST, else the two heaps with the id filter and tombstones as the "allowed" test and hnswlib's strict stop rule
// whenever anything is filtered out.  Emits the k best ascending by (distance, label).
template <bool L2, bool FAST>
__global__ void __launch_bounds__(HNSW_THREADS) hnsw_search_kernel(const HnswDev g, const float* __restrict__ queries, long long nq,
                                                                  int k, int ef, FilterDev filt, unsigned int* visited /*[nq, words]*/,
                                                                  long long words, HeapEnt* cand_pool, long long cand_cap, float* out_dist,
                                                                  long long* out_ids) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ float s_d[32];
  __shared__ unsigned int s_id[32];
  __shared__ int s_m;
  const long long qi = blockIdx.x;
  const int d = g.d;
  float* qs = reinterpret_cast<float*>(smem);
  HeapEnt* top_sm = reinterpret_cast<HeapEnt*>(smem + walk_qbytes(d));                                      // [ef + 1]
  HeapEnt* cand_sm = reinterpret_cast<HeapEnt*>(smem + walk_qbytes(d) + (size_t)(ef + 1) * sizeof(HeapEnt));  // [HNSW_CAND_SMEM]
  for (int i = threadIdx.x; i < d; i += HNSW_THREADS) qs[i] = queries[(size_t)qi * d + i];
  if (g.n == 0) {
    for (int i = threadIdx.x; i < k; i += HNSW_THREADS) { out_dist[(size_t)qi * k + i] = 0.f; out_ids[(size_t)qi * k + i] = -1; }
    return;
  }
  __syncthreads();
  const Walk<L2> w{g, qs, visited + (size_t)qi * words, s_d, s_id, &s_m, d, (int)threadIdx.x >> 2, (int)threadIdx.x & 3, (d & 3) == 0};
  unsigned int cur = g.enterpoint;
  float curdist = w.score_one(cur);
  descend(w, g.maxlevel, 0, cur, curdist);
  if (FAST) {
    HeapEnt* T = top_sm;
    const int ntop = walk_merged(w, 0, ef, cur, curdist, T, cand_sm);  // HNSW_CAND_SMEM >= ef + 1 is checked on the host
    if (threadIdx.x == 0) {  // emit the k best ascending by (distance, label)
      const int have = min(ntop, k);
      for (int i = 0; i < have; ++i) {
        int best = i;
        for (int j = i + 1; j < ntop && T[j].d == T[i].d; ++j)  // equal distances: smaller label first (T is ascending in d)
          if (g.labels[T[j].id & 0x7fffffffu] < g.labels[T[best].id & 0x7fffffffu]) best = j;
        const HeapEnt tmp = T[i]; T[i] = T[best]; T[best] = tmp;
        out_dist[(size_t)qi * k + i] = T[i].d;
        out_ids[(size_t)qi * k + i] = g.labels[T[i].id & 0x7fffffffu];
      }
      for (int i = have; i < k; ++i) { out_dist[(size_t)qi * k + i] = 0.f; out_ids[(size_t)qi * k + i] = -1; }
    }
    return;
  }
  const HeapRef top{top_sm, top_sm, ef + 1};
  const HeapRef cand{cand_sm, cand_pool + (size_t)qi * cand_cap, HNSW_CAND_SMEM};
  const bool strict_stop = filt.has_range || filt.sorted_ids != nullptr || g.has_deletions;
  int ntop = walk_heaps(w, 0, ef, strict_stop, [&](unsigned int c) { return !g.deleted[c] && filter_pass(filt, g.labels[c]); },
                        cur, curdist, top, cand);
  if (threadIdx.x == 0) {
    // keep the k best, emit ascending by (distance, label)
    while (ntop > k) h_pop<true>(top, ntop);
    for (int i = 0; i < ntop; ++i) {  // selection sort of <= k entries
      int best = i;
      for (int j = i + 1; j < ntop; ++j) {
        const long long lj = g.labels[top_sm[j].id], lb = g.labels[top_sm[best].id];
        if (top_sm[j].d < top_sm[best].d || (top_sm[j].d == top_sm[best].d && lj < lb)) best = j;
      }
      const HeapEnt tmp = top_sm[i]; top_sm[i] = top_sm[best]; top_sm[best] = tmp;
      out_dist[(size_t)qi * k + i] = top_sm[i].d;
      out_ids[(size_t)qi * k + i] = g.labels[top_sm[i].id];
    }
    for (int i = ntop; i < k; ++i) { out_dist[(size_t)qi * k + i] = 0.f; out_ids[(size_t)qi * k + i] = -1; }
  }
}

// ---------------- batched construction on the device (DESIGN §4.4) ----------------
// A batch of rows is inserted against the graph as it was at the batch start: construction search per (row, level), then
// forward links per (row, level) from the search result plus the batch's earlier rows, then reverse links grouped per
// (level, target).  Candidate lists are ordered by the 64-bit key ord(distance) << 32 | node id, so every tie is broken by
// insertion index and nothing depends on thread timing.
constexpr int HNSW_BUILD_MAX_BATCH = 8192;  // rows per batch (the peer matrix is batch^2 floats)
constexpr int HNSW_BUILD_DEFAULT_BATCH = 2048;

__device__ __forceinline__ unsigned long long cand_key(float d, unsigned int id) { return ((unsigned long long)f2ord(d) << 32) | id; }

// ascending sort of keys[0, p2) (p2 a power of two), all threads of the CTA
__device__ void bitonic_sort(unsigned long long* keys, int p2) {
  __syncthreads();
  for (int k = 2; k <= p2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int x = threadIdx.x; x < p2; x += HNSW_THREADS) {
        const int y = x ^ j;
        if (y > x) {
          const unsigned long long a = keys[x], b = keys[y];
          if ((a > b) == ((x & k) == 0)) { keys[x] = b; keys[y] = a; }
        }
      }
      __syncthreads();
    }
}

// HostGraph::heuristic over the ascending candidates C[0, c): keeps a candidate unless a node already kept is closer to it
// than the base; fewer than lim candidates are all kept.  sel[0, return) ascending.  All 32 quads score one candidate against
// up to 32 kept nodes per round.
template <bool L2>
__device__ int heuristic_select(const unsigned long long* C, int c, int lim, unsigned int* sel, const float* data, int d) {
  __syncthreads();
  if (c < lim) {
    for (int i = threadIdx.x; i < c; i += HNSW_THREADS) sel[i] = (unsigned int)C[i];
    __syncthreads();
    return c;
  }
  const int quad = threadIdx.x >> 2, t = threadIdx.x & 3;
  const bool vec = (d & 3) == 0;
  int nsel = 0;
  for (int k = 0; k < c && nsel < lim; ++k) {
    const unsigned int cand = (unsigned int)C[k];
    const float dq = ord2f((unsigned int)(C[k] >> 32));
    bool bad = false;
    for (int s0 = 0; s0 < nsel; s0 += 32) {
      const int s = s0 + quad;
      const float v = hnsw_distance<L2>(data + (size_t)sel[s < nsel ? s : 0] * d, data + (size_t)cand * d, d, t, vec);
      if (s < nsel && v < dq) bad = true;
    }
    if (!__syncthreads_or(bad)) {
      if (threadIdx.x == 0) sel[nsel] = cand;
      ++nsel;
      __syncthreads();
    }
  }
  return nsel;
}

// Construction search: one CTA per batch row r, whose vector is node g.n + r.  Greedy descent from the entry point through
// the levels above the row's own, then HostGraph::search_layer with ef = efc at every level from min(level, maxlevel) down to
// 0, each starting from the closest node found one level up.  out[(slot_off[r] + l) * efc ...] = the result at level l,
// ascending by (distance, node); out_cnt = its length.  FAST = no tombstones and efc + 1 <= HNSW_CAND_SMEM: the merged-array
// form; otherwise the two heaps with tombstones as the "allowed" test and the strict stop rule.  The visited bitset is
// cleared per level.
template <bool L2, bool FAST>
__global__ void __launch_bounds__(HNSW_THREADS) hnsw_build_search_kernel(const HnswDev g, const int* __restrict__ levels, long long row0,
                                                                        const long long* __restrict__ slot_off, unsigned int* visited,
                                                                        long long words, HeapEnt* cand_pool, long long cand_cap, HeapEnt* out,
                                                                        int* out_cnt) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ float s_d[32];
  __shared__ unsigned int s_id[32];
  __shared__ int s_m;
  __shared__ unsigned int s_cur;
  __shared__ float s_curdist;
  const long long r = row0 + blockIdx.x;
  const int d = g.d, efc = g.efc;
  float* qs = reinterpret_cast<float*>(smem);
  HeapEnt* top_sm = reinterpret_cast<HeapEnt*>(smem + walk_qbytes(d));
  HeapEnt* cand_sm = top_sm + efc + 1;
  for (int i = threadIdx.x; i < d; i += HNSW_THREADS) qs[i] = g.data[(size_t)(g.n + r) * d + i];
  __syncthreads();
  const Walk<L2> w{g, qs, visited + (size_t)blockIdx.x * words, s_d, s_id, &s_m, d, (int)(threadIdx.x >> 2), (int)(threadIdx.x & 3), (d & 3) == 0};
  const int lev = levels[r];
  unsigned int cur = g.enterpoint;
  float curdist = w.score_one(cur);
  descend(w, g.maxlevel, lev, cur, curdist);  // (add_point: only when the row's level is below maxlevel)
  for (int level = min(lev, g.maxlevel); level >= 0; --level) {
    __syncthreads();
    for (long long x = threadIdx.x; x < words; x += HNSW_THREADS) w.vis[x] = 0u;
    __syncthreads();
    HeapEnt* res = out + (size_t)(slot_off[r] + level) * efc;
    if (FAST) {
      HeapEnt* T = top_sm;
      const int ntop = walk_merged(w, level, efc, cur, curdist, T, cand_sm);
      if (threadIdx.x == 0) {  // T is ascending in distance; equal distances go by node id
        for (int i = 0; i < ntop; ++i) {
          HeapEnt e = T[i];
          e.id &= 0x7fffffffu;
          int j = i;
          while (j > 0 && res[j - 1].d == e.d && res[j - 1].id > e.id) { res[j] = res[j - 1]; --j; }
          res[j] = e;
        }
        out_cnt[slot_off[r] + level] = ntop;
        if (ntop > 0) { s_cur = res[0].id; s_curdist = res[0].d; }
      }
    } else {
      const HeapRef top{top_sm, top_sm, efc + 1};
      const HeapRef cand{cand_sm, cand_pool + (size_t)blockIdx.x * cand_cap, HNSW_CAND_SMEM};
      int ntop = walk_heaps(w, level, efc, true, [&](unsigned int c) { return !g.deleted[c]; }, cur, curdist, top, cand);
      if (threadIdx.x == 0) {
        const int cnt = ntop;
        while (ntop > 0) { const HeapEnt e = top.get(0); h_pop<true>(top, ntop); res[ntop] = e; }  // largest first -> ascending
        for (int i = 1; i < cnt; ++i) {
          const HeapEnt e = res[i];
          int j = i;
          while (j > 0 && res[j - 1].d == e.d && res[j - 1].id > e.id) { res[j] = res[j - 1]; --j; }
          res[j] = e;
        }
        out_cnt[slot_off[r] + level] = cnt;
        if (cnt > 0) { s_cur = res[0].id; s_curdist = res[0].d; }
      }
    }
    if (threadIdx.x == 0 && out_cnt[slot_off[r] + level] == 0) { s_cur = cur; s_curdist = curdist; }
    __syncthreads();
    cur = s_cur;
    curdist = s_curdist;
  }
}

// Peer distances of a batch: peer[i * nb + j] for j < i only (the link kernel reads no other entry), one quad per pair, in
// pair_distance_kernel's arithmetic (hnsw_distance).
template <bool L2>
__global__ void __launch_bounds__(256) hnsw_peer_distance_kernel(const float* __restrict__ rows, int nb, int d, float* __restrict__ peer) {
  const long long pair = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
  const int t = threadIdx.x & 3;
  const long long total = (long long)nb * (nb - 1) / 2;
  const bool valid = pair < total;
  const long long p = valid ? pair : 0;
  long long i = (long long)((1.0 + sqrt(1.0 + 8.0 * (double)p)) / 2.0);  // p = i (i - 1) / 2 + j, 0 <= j < i
  while (i * (i - 1) / 2 > p) --i;
  while ((i + 1) * i / 2 <= p) ++i;
  const long long j = p - i * (i - 1) / 2;
  const float v = hnsw_distance<L2>(rows + (size_t)i * d, rows + (size_t)j * d, d, t, (d & 3) == 0);
  if (valid && t == 0) peer[(size_t)i * nb + j] = v;
}

// deleted[ids[k]] = 1: the tombstones of one batch in one launch
__global__ void hnsw_tombstone_kernel(unsigned char* deleted, const unsigned int* __restrict__ ids, long long n) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) deleted[ids[k]] = 1;
}

// Forward links: one CTA per (row, level) task.  Candidates = the search result at that level merged with the batch's earlier
// rows j < i whose level reaches it (peer distances from the pair matrix), best efc by key; heuristic(M) of those is written
// farthest first, as HostGraph::connect writes it.  Each kept target t emits the reverse-link key (level, t, i) into
// trip[task * M + s]; unused slots hold ~0.
template <bool L2>
__global__ void __launch_bounds__(HNSW_THREADS) hnsw_build_link_kernel(const HnswDev b, long long n0, int nb, const int* __restrict__ levels,
                                                                      int maxlevel, const float* __restrict__ peer, const long long* __restrict__ slot_off,
                                                                      const HeapEnt* __restrict__ sres, const int* __restrict__ scnt,
                                                                      const int2* __restrict__ tasks, unsigned long long* trip) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int s_cp;
  const int2 task = tasks[blockIdx.x];
  const int i = task.x, l = task.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem);
  const int top_level = min(levels[i], maxlevel);
  const long long slot = slot_off[i] + l;
  const int cs = l <= top_level ? scnt[slot] : 0;
  for (int k = threadIdx.x; k < cs; k += HNSW_THREADS) keys[k] = cand_key(sres[(size_t)slot * b.efc + k].d, sres[(size_t)slot * b.efc + k].id);
  __syncthreads();
  // a peer can only enter a full list below its last key (peer ids are larger than every graph node's)
  const unsigned long long tau = cs == b.efc ? keys[cs - 1] : ~0ull;
  if (warp == 0) {
    int cp = 0;
    for (int j0 = 0; j0 < i; j0 += 32) {
      const int j = j0 + lane;
      unsigned long long key = ~0ull;
      if (j < i && levels[j] >= l) key = cand_key(peer[(size_t)i * nb + j], (unsigned int)(n0 + j));
      const bool ok = key < tau;
      const unsigned int mask = __ballot_sync(0xffffffffu, ok);
      if (ok) keys[cs + cp + __popc(mask & ((1u << lane) - 1u))] = key;
      cp += __popc(mask);
    }
    if (lane == 0) s_cp = cp;
  }
  __syncthreads();
  int c = cs + s_cp;
  if (s_cp > 0) {
    int p2 = 1;
    while (p2 < c) p2 <<= 1;
    for (int k = c + threadIdx.x; k < p2; k += HNSW_THREADS) keys[k] = ~0ull;
    bitonic_sort(keys, p2);
    c = min(c, b.efc);
  }
  unsigned int* sel = reinterpret_cast<unsigned int*>(smem + (size_t)(b.efc + nb) * 2 * sizeof(unsigned long long));
  const int nsel = heuristic_select<L2>(keys, c, b.M, sel, b.data, b.d);
  unsigned int* list = b.links((unsigned int)(n0 + i), l);
  for (int s = threadIdx.x; s < nsel; s += HNSW_THREADS) list[1 + s] = sel[nsel - 1 - s];
  if (threadIdx.x == 0) list[0] = (unsigned int)nsel;
  for (int s = threadIdx.x; s < b.M; s += HNSW_THREADS)
    trip[(size_t)blockIdx.x * b.M + s] = s < nsel ? ((unsigned long long)l << 52) | ((unsigned long long)sel[s] << 20) | (unsigned long long)i : ~0ull;
}

// Reverse links: keys sorted ascending group the sources of every (level, target) in call order.  The CTA of a group's first
// key appends the sources when they fit into the target's list, and otherwise rewrites the list as heuristic(list ∪ sources,
// Mmax) farthest first (connect's shrink).  Entries past the new size keep their old values, as in connect.
template <bool L2>
__global__ void __launch_bounds__(HNSW_THREADS) hnsw_build_reverse_kernel(const HnswDev b, long long n0, const unsigned long long* __restrict__ keys,
                                                                         long long total) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int s_ns;
  const long long k0 = blockIdx.x;
  const unsigned long long key = keys[k0];
  if (key == ~0ull) return;
  if (k0 > 0 && (keys[k0 - 1] >> 20) == (key >> 20)) return;
  if (threadIdx.x == 0) {
    long long e = k0 + 1;
    while (e < total && (keys[e] >> 20) == (key >> 20)) ++e;
    s_ns = (int)(e - k0);
  }
  __syncthreads();
  const int ns = s_ns;
  const int l = (int)(key >> 52);
  const unsigned int tgt = (unsigned int)((key >> 20) & 0xffffffffu);
  const int mcur = l ? b.maxM : b.maxM0;
  unsigned int* list = b.links(tgt, l);
  const int sz = (int)list[0];
  auto source = [&](int s) { return (unsigned int)(n0 + (long long)(keys[k0 + s] & 0xfffffu)); };
  if (sz + ns <= mcur) {
    for (int s = threadIdx.x; s < ns; s += HNSW_THREADS) list[1 + sz + s] = source(s);
    __syncthreads();
    if (threadIdx.x == 0) list[0] = (unsigned int)(sz + ns);
    return;
  }
  unsigned long long* cand = reinterpret_cast<unsigned long long*>(smem);
  const int c = sz + ns;
  int p2 = 1;
  while (p2 < c) p2 <<= 1;
  unsigned int* sel = reinterpret_cast<unsigned int*>(smem + (size_t)p2 * sizeof(unsigned long long));
  const int quad = threadIdx.x >> 2, t = threadIdx.x & 3;
  const bool vec = (b.d & 3) == 0;
  for (int c0 = 0; c0 < p2; c0 += 32) {
    const int x = c0 + quad;
    const unsigned int id = x < sz ? list[1 + x] : x < c ? source(x - sz) : tgt;
    const float v = hnsw_distance<L2>(b.data + (size_t)id * b.d, b.data + (size_t)tgt * b.d, b.d, t, vec);
    if (t == 0 && x < p2) cand[x] = x < c ? cand_key(v, id) : ~0ull;
  }
  bitonic_sort(cand, p2);
  const int nsel = heuristic_select<L2>(cand, c, mcur, sel, b.data, b.d);
  for (int s = threadIdx.x; s < nsel; s += HNSW_THREADS) list[1 + s] = sel[nsel - 1 - s];
  if (threadIdx.x == 0) list[0] = (unsigned int)nsel;
}

// NormalizeVectorForHnsw (vector_index_utils.cc:493-500): the row cosine stores and searches, o = x / (|x| + 1e-30)
void normalize_for_hnsw(const float* x, int d, float* o) {
  float norm = 0.0f;
  for (int j = 0; j < d; ++j) norm += x[j] * x[j];
  norm = 1.0f / (sqrtf(norm) + 1e-30f);
  for (int j = 0; j < d; ++j) o[j] = x[j] * norm;
}

// f(L2, FAST), both as std::integral_constant: the one place a walk kernel's instantiation is chosen
template <class F>
void dispatch_walk(bool l2, bool fast, F&& f) {
  if (l2) { if (fast) f(std::true_type(), std::true_type()); else f(std::true_type(), std::false_type()); }
  else { if (fast) f(std::false_type(), std::true_type()); else f(std::false_type(), std::false_type()); }
}

}  // namespace

struct HnswIndex : IndexBase {
  HostGraph G;
  int64_t max_element_limit;
  int ef = 10;  // hnswlib default; sticky setEf (hnsw.cc:426-428)
  bool dirty = true;
  int64_t uploaded_rows = 0;
  DevBuf<float> d_data;
  DevBuf<long long> d_labels;
  DevBuf<int64_t> d_upoff;
  DevBuf<unsigned int> d_link0, d_linkup;
  DevBuf<unsigned char> d_deleted;

  // the device mirror as the kernels see it: its first n nodes, entered at ep on level maxlevel
  HnswDev dev_graph(long long n, int maxlevel, tableint ep, bool deletions) const {
    HnswDev g;
    g.data = d_data.p; g.labels = d_labels.p; g.link0 = d_link0.p; g.up_off = d_upoff.p; g.linkup = d_linkup.p; g.deleted = d_deleted.p;
    g.n = n; g.d = dim; g.M = (int)G.M; g.maxM = (int)G.maxM; g.maxM0 = (int)G.maxM0; g.efc = (int)G.efc;
    g.maxlevel = maxlevel; g.enterpoint = ep; g.has_deletions = deletions;
    return g;
  }

  HnswIndex(b200vs_metric m, int d, const b200vs_params& p) : IndexBase(B200VS_HNSW, m, d, p) {
    if (p.hnsw_m <= 0 || p.hnsw_efc <= 0) fail(B200VS_EILLEGAL_PARAMETERS, "hnsw nlinks / efconstruction must be > 0");
    max_element_limit = p.max_elements > 0 ? p.max_elements : (1LL << 40);
    G.init(metric, d, p.hnsw_m, p.hnsw_efc, 100);  // random_seed = 100, hnsw.cc:181-182
  }

  void set_state(const void* blob, size_t len) override {
    std::unique_lock<std::shared_mutex> wl(rw);
    G = parse_state(G, blob, len);
    dirty = true; uploaded_rows = 0;
  }

  // VectorIndexHnsw::Upsert, hnsw.cc:203-254 (Add == Upsert; vectors are normalised per row for cosine).  The builders take
  // host rows: device rows are downloaded first.  batched: b200vs_hnsw_add_batched.
  void add(const AddReq& r) override {
    WriteHold hold(this);
    std::vector<float> hx;
    std::vector<int64_t> hid;
    const float* x = static_cast<const float*>(r.x);
    const int64_t* ids = r.ids;
    if (r.on_device) {
      hx.resize((size_t)r.n * dim);
      B200VS_CUDA(cudaMemcpyAsync(hx.data(), x, hx.size() * 4, cudaMemcpyDeviceToHost, stream));
      if (!ids) {
        hid.resize(r.n);
        B200VS_CUDA(cudaMemcpyAsync(hid.data(), r.ids_dev, (size_t)r.n * 8, cudaMemcpyDeviceToHost, stream));
        ids = hid.data();
      }
      B200VS_CUDA(cudaStreamSynchronize(stream));
      x = hx.data();
    }
    check_ids_nonnegative(r.n, ids);
    if (r.batched) add_batched_locked(r.n, x, ids, r.batch, r.form != AddReq::RAW);
    else add_host_locked(r.n, x, ids, r.form != AddReq::RAW);
  }
  // the host builder with the writer hold taken; prepared = rows stored as given (cosine rows are already normalised)
  void add_host_locked(int64_t n, const float* x, const int64_t* in_ids, bool is_prepared) {
    if (G.n + n > max_element_limit) fail(B200VS_EINTERNAL, "upsert failed, exceeds max elements");
    auto prepared = [&](int64_t i, std::vector<float>& tmp) -> const float* {
      const float* xi = x + (size_t)i * dim;
      if (metric != B200VS_COSINE || is_prepared) return xi;
      normalize_for_hnsw(xi, dim, tmp.data());
      return tmp.data();
    };
    // every slot of the call up front: node c takes the generator's c-th draw, as when each insertion drew its own level
    const int64_t ntot = G.n + n;
    G.append_nodes(G.draw_levels(n, G.rng));
    const int nthreads = (int)std::min<int64_t>(std::max(1, params.hnsw_build_threads), n);
    if (nthreads <= 1) {  // single writer: deterministic graph (equal to the oracle's for the same insertion order)
      std::vector<float> tmp(dim);
      for (int64_t i = 0; i < n; ++i) G.add_point<false>(prepared(i, tmp), in_ids[i]);
    } else {  // concurrent insertion, as the reference's thread pool does (hnsw.cc:229-243)
      G.reserve_locks(ntot);
      std::atomic<int64_t> next{0};
      if (G.n == 0) { std::vector<float> tmp(dim); G.add_point<false>(prepared(0, tmp), in_ids[0]); next = 1; }  // hnswlib: first element alone
      std::vector<std::thread> ts;
      for (int t = 0; t < nthreads; ++t)
        ts.emplace_back([&]() {
          HostGraph::VisitCtx vc;
          vc.visited.assign((size_t)ntot, 0u);
          std::vector<float> tmp(dim);
          for (;;) {
            const int64_t i = next.fetch_add(1);
            if (i >= n) break;
            G.add_point<true>(prepared(i, tmp), in_ids[i], &vc);
          }
        });
      for (auto& th : ts) th.join();
    }
    dirty = true;
  }
  // add's refusals (batched: the batched build's, for that batch size), which come before either changes anything
  void check_add(const AddReq& r) override {
    IndexBase::check_add(r);
    RwSharedGuard rl(this);
    if (r.batched) batched_plan(r.n, r.batch);
    else if (G.n + r.n > max_element_limit) fail(B200VS_EINTERNAL, "upsert failed, exceeds max elements");
  }
  // b200vs_hnsw_add_batched: the rule of DESIGN §4.4.  The host plans every batch first on a copy of the bookkeeping it needs
  // (levels from a copy of G.rng in call order, the batch schedule, tombstones, node ids, entry point); the device mirror then
  // builds the links batch after batch in stream order.  G (and its generator) changes only once the device work has
  // finished: a call that fails on the way leaves the index as it was and marks the mirror for a full re-upload.
  int64_t build_scratch_limit = 0;  // b200vs_debug_hnsw_build_scratch_limit: device scratch bytes one call may take, 0 = no cap

  // the batch size and the construction kernels' shared memory of the batched build of n rows, after its refusals
  struct BuildPlan { int batch, bmax; size_t smem_search, smem_link, smem_rev; };
  BuildPlan batched_plan(int64_t n, int batch) const {
    if (G.n + n > max_element_limit) fail(B200VS_EINTERNAL, "upsert failed, exceeds max elements");
    if (G.n + n >= (1LL << 31)) fail(B200VS_EILLEGAL_PARAMETERS, "batched HNSW construction holds at most 2^31 - 1 nodes");
    BuildPlan P;
    P.batch = batch <= 0 ? HNSW_BUILD_DEFAULT_BATCH : std::min(batch, HNSW_BUILD_MAX_BATCH);
    P.bmax = (int)std::min<int64_t>(P.batch, n);  // largest batch of this call
    P.smem_search = walk_smem_bytes(dim, (int)G.efc);
    P.smem_link = (size_t)((int)G.efc + P.bmax) * 2 * sizeof(unsigned long long) + (size_t)G.M * 4;
    P.smem_rev = (size_t)((int)G.maxM0 + P.bmax) * 2 * sizeof(unsigned long long) + (size_t)G.maxM0 * 4;
    if (P.smem_search > HNSW_SMEM_LIMIT || P.smem_link > HNSW_SMEM_LIMIT || P.smem_rev > HNSW_SMEM_LIMIT)
      fail(B200VS_EILLEGAL_PARAMETERS, "efconstruction / dimension / batch too large for the batched construction kernels");
    return P;
  }

  // the batched build with the writer hold taken; prepared = rows stored as given (cosine rows are already normalised)
  void add_batched_locked(int64_t n, const float* x, const int64_t* in_ids, int batch, bool prepared) {
    const BuildPlan P = batched_plan(n, batch);
    batch = P.batch;
    const int efc = (int)G.efc, M = (int)G.M, maxM0 = (int)G.maxM0;
    const int bmax = P.bmax;
    const size_t smem_search = P.smem_search;
    cudaStream_t s = stream;
    upload(s);

    // ---- plan (host), on copies: G is not touched until the device work is done ----
    const int64_t n0_call = G.n, ntot = G.n + n;
    std::vector<float> rows((size_t)n * dim);
    for (int64_t i = 0; i < n; ++i) {
      if (metric == B200VS_COSINE && !prepared) normalize_for_hnsw(x + (size_t)i * dim, dim, &rows[(size_t)i * dim]);
      else memcpy(&rows[(size_t)i * dim], x + (size_t)i * dim, (size_t)dim * 4);
    }
    std::default_random_engine rng = G.rng;
    const std::vector<int> lev = G.draw_levels(n, rng);
    struct Batch { int64_t a, b; int maxlevel; tableint ep; bool deletions; int64_t task0, ntask, dead0, ndead; };
    std::vector<Batch> plan;
    std::vector<long long> slot_off(n);
    std::vector<int2> tasks;
    std::vector<unsigned int> dead;               // nodes tombstoned at each batch start (Batch::dead0, ndead)
    std::unordered_map<int64_t, tableint> fresh;  // labels inserted by this call -> their latest node (live)
    int64_t gn = G.n, ndel = G.ndeleted;
    int maxlevel = G.maxlevel;
    tableint ep = G.enterpoint;
    int64_t max_slots = 0;
    std::unordered_set<int64_t> in_batch;
    for (int64_t a = 0; a < n;) {
      Batch B;
      B.a = a;
      const int64_t lim = gn == 0 ? 1 : std::min<int64_t>(batch, gn);
      in_batch.clear();
      int64_t e = a;
      while (e < n && e - a < lim && in_batch.insert(in_ids[e]).second) ++e;
      B.b = e;
      B.dead0 = (int64_t)dead.size();
      for (int64_t i = a; i < e; ++i) {  // add_point's tombstone of a label already present
        auto f = fresh.find(in_ids[i]);
        if (f != fresh.end()) { dead.push_back(f->second); continue; }
        auto it = G.lookup.find(in_ids[i]);
        if (it != G.lookup.end() && !G.deleted[it->second]) dead.push_back(it->second);
      }
      B.ndead = (int64_t)dead.size() - B.dead0;
      ndel += B.ndead;
      B.maxlevel = maxlevel; B.ep = ep; B.deletions = ndel > 0;
      B.task0 = (int64_t)tasks.size();
      long long slots = 0;
      for (int64_t i = a; i < e; ++i) {
        fresh[in_ids[i]] = (tableint)(gn++);
        slot_off[i] = slots;
        slots += std::min(lev[i], B.maxlevel) + 1;
        for (int l = 0; l <= lev[i]; ++l) tasks.push_back(make_int2((int)(i - a), l));
      }
      max_slots = std::max<int64_t>(max_slots, slots);
      B.ntask = (int64_t)tasks.size() - B.task0;
      for (int64_t i = a; i < e; ++i)  // entry point in call order
        if (lev[i] > maxlevel) { ep = (tableint)(n0_call + i); maxlevel = lev[i]; }
      plan.push_back(B);
      a = e;
    }
    std::vector<int64_t> off{G.up_off[n0_call]};  // the call's nodes' pool offsets
    G.extend_up_off(off, lev);
    const int64_t up_old = off[0], up_new = off[n];
    std::vector<tableint> up((size_t)up_new), l0((size_t)ntot * (maxM0 + 1));  // the link lists coming back from the device

    try {
      // ---- device mirror: append the call's rows, empty link lists and upper-level slots (beyond G.n: unseen by searches) ----
      d_data.reserve((size_t)ntot * dim, (size_t)n0_call * dim, s);
      d_labels.reserve(ntot, n0_call, s); d_deleted.reserve(ntot, n0_call, s); d_upoff.reserve(ntot + 1, n0_call, s);
      d_link0.reserve((size_t)ntot * (maxM0 + 1), (size_t)n0_call * (maxM0 + 1), s);
      d_linkup.reserve((size_t)std::max<long long>(up_new, 1), (size_t)up_old, s);
      B200VS_CUDA(cudaMemcpyAsync(d_data.p + (size_t)n0_call * dim, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, s));
      B200VS_CUDA(cudaMemcpyAsync(d_labels.p + n0_call, in_ids, (size_t)n * 8, cudaMemcpyHostToDevice, s));
      B200VS_CUDA(cudaMemsetAsync(d_deleted.p + n0_call, 0, (size_t)n, s));
      B200VS_CUDA(cudaMemcpyAsync(d_upoff.p + n0_call, off.data(), (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, s));
      B200VS_CUDA(cudaMemsetAsync(d_link0.p + (size_t)n0_call * (maxM0 + 1), 0, (size_t)n * (maxM0 + 1) * 4, s));
      if (up_new > up_old) B200VS_CUDA(cudaMemsetAsync(d_linkup.p + up_old, 0, (size_t)(up_new - up_old) * 4, s));

      // ---- scratch, freed at the end of the call ----
      size_t scratch_bytes = 0;
      auto take = [&](auto& buf, size_t count) {  // a device reservation counted against build_scratch_limit
        if (count <= buf.cap) return;
        const size_t after = scratch_bytes + (count - buf.cap) * sizeof(*buf.p);
        if (build_scratch_limit > 0 && after > (size_t)build_scratch_limit)
          throw CudaError("HNSW batched construction: device scratch over the limit (out of memory)");
        buf.reserve(count, 0, s);  // a grown buffer needs none of its old contents
        scratch_bytes = after;
      };
      const bool any_heap = efc + 1 > HNSW_CAND_SMEM || std::any_of(plan.begin(), plan.end(), [](const Batch& B) { return B.deletions; });
      const long long words_max = (ntot + 31) / 32;
      const size_t row_bytes = (size_t)words_max * 4 + (any_heap ? (size_t)(ntot + 1) * sizeof(HeapEnt) : 0);
      const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(bmax, (int64_t)(HNSW_CAND_POOL_BYTES / row_bytes)));
      int64_t max_task = 1;
      for (const Batch& B : plan) max_task = std::max(max_task, B.ntask);
      const size_t ntrip = (size_t)max_task * M;
      DevBuf<unsigned int> d_vis, d_dead;
      DevBuf<HeapEnt> d_pool, d_sres;
      DevBuf<int> d_scnt, d_lev;
      DevBuf<long long> d_slot;
      DevBuf<int2> d_tasks;
      DevBuf<float> d_peer;  // grows with the batches (1, 1, 2, 4, ... rows)
      DevBuf<unsigned long long> d_trip, d_trip_sorted;
      DevBuf<unsigned char> d_sort;
      take(d_vis, (size_t)chunk * words_max);
      if (any_heap) take(d_pool, (size_t)chunk * (ntot + 1));
      take(d_sres, (size_t)std::max<int64_t>(max_slots, 1) * efc);
      take(d_scnt, (size_t)std::max<int64_t>(max_slots, 1));
      take(d_lev, (size_t)n);
      take(d_slot, (size_t)n);
      take(d_tasks, std::max<size_t>(tasks.size(), 1));
      take(d_dead, std::max<size_t>(dead.size(), 1));
      take(d_trip, ntrip); take(d_trip_sorted, ntrip);
      size_t sort_bytes = 0;
      B200VS_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, sort_bytes, d_trip.p, d_trip_sorted.p, (int)ntrip, 0, 64, s));
      take(d_sort, std::max<size_t>(sort_bytes, 1));
      B200VS_CUDA(cudaMemcpyAsync(d_lev.p, lev.data(), (size_t)n * 4, cudaMemcpyHostToDevice, s));
      B200VS_CUDA(cudaMemcpyAsync(d_slot.p, slot_off.data(), (size_t)n * 8, cudaMemcpyHostToDevice, s));
      if (!tasks.empty()) B200VS_CUDA(cudaMemcpyAsync(d_tasks.p, tasks.data(), tasks.size() * sizeof(int2), cudaMemcpyHostToDevice, s));
      if (!dead.empty()) B200VS_CUDA(cudaMemcpyAsync(d_dead.p, dead.data(), dead.size() * 4, cudaMemcpyHostToDevice, s));

      const bool l2 = metric == B200VS_L2;
      auto setsmem = [](const void* fn) { B200VS_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)HNSW_SMEM_LIMIT)); };
      for (const bool fast : {true, false})
        dispatch_walk(l2, fast, [&](auto L2_, auto FAST_) { setsmem((const void*)hnsw_build_search_kernel<decltype(L2_)::value, decltype(FAST_)::value>); });
      if (l2) { setsmem((const void*)hnsw_build_link_kernel<true>); setsmem((const void*)hnsw_build_reverse_kernel<true>); }
      else { setsmem((const void*)hnsw_build_link_kernel<false>); setsmem((const void*)hnsw_build_reverse_kernel<false>); }
      if (profiling) for (int p = PH_BUILD_SEARCH; p <= PH_BUILD_LINK; ++p) phase_ms[p] = 0.f;
      for (const Batch& B : plan) {
        if (B.ndead > 0) {
          hnsw_tombstone_kernel<<<(unsigned)cdiv(B.ndead, 256), 256, 0, s>>>(d_deleted.p, d_dead.p + B.dead0, B.ndead);
          B200VS_CUDA(cudaGetLastError());
        }
        const long long n0 = n0_call + B.a;
        const int nb = (int)(B.b - B.a);
        if (n0 == 0) continue;  // the first row of an empty graph goes in alone, without links
        if (nb > 1) take(d_peer, (size_t)nb * nb);
        const HnswDev g = dev_graph(n0, B.maxlevel, B.ep, B.deletions);
        const bool fast = !B.deletions && efc + 1 <= HNSW_CAND_SMEM;
        const long long words = (n0 + 31) / 32, cand_cap = fast ? 0 : n0 + 1;
        phase(PH_BUILD_SEARCH, s);
        dispatch_walk(l2, fast, [&](auto L2_, auto FAST_) {
          const auto kernel = hnsw_build_search_kernel<decltype(L2_)::value, decltype(FAST_)::value>;
          for (int64_t r0 = 0; r0 < nb; r0 += chunk) {
            const unsigned m = (unsigned)std::min<int64_t>(chunk, nb - r0);
            kernel<<<m, HNSW_THREADS, smem_search, s>>>(g, d_lev.p + B.a, r0, d_slot.p + B.a, d_vis.p, words, d_pool.p, cand_cap, d_sres.p,
                                                       d_scnt.p);
            B200VS_CUDA(cudaGetLastError());
          }
        });
        phase(PH_BUILD_SELECT, s);
        if (nb > 1) {
          const unsigned grid = (unsigned)cdiv((int64_t)nb * (nb - 1) / 2 * 4, 256);
          const float* brows = d_data.p + (size_t)n0 * dim;
          if (l2) hnsw_peer_distance_kernel<true><<<grid, 256, 0, s>>>(brows, nb, dim, d_peer.p);
          else hnsw_peer_distance_kernel<false><<<grid, 256, 0, s>>>(brows, nb, dim, d_peer.p);
          B200VS_CUDA(cudaGetLastError());
        }
        const size_t smem_l = (size_t)(efc + nb) * 2 * sizeof(unsigned long long) + (size_t)M * 4;
        if (l2) hnsw_build_link_kernel<true><<<(unsigned)B.ntask, HNSW_THREADS, smem_l, s>>>(g, n0, nb, d_lev.p + B.a, B.maxlevel, d_peer.p, d_slot.p + B.a, d_sres.p, d_scnt.p, d_tasks.p + B.task0, d_trip.p);
        else hnsw_build_link_kernel<false><<<(unsigned)B.ntask, HNSW_THREADS, smem_l, s>>>(g, n0, nb, d_lev.p + B.a, B.maxlevel, d_peer.p, d_slot.p + B.a, d_sres.p, d_scnt.p, d_tasks.p + B.task0, d_trip.p);
        B200VS_CUDA(cudaGetLastError());
        phase(PH_BUILD_LINK, s);
        const int nt = (int)(B.ntask * M);
        size_t tb = sort_bytes;
        B200VS_CUDA(cub::DeviceRadixSort::SortKeys(d_sort.p, tb, d_trip.p, d_trip_sorted.p, nt, 0, 64, s));
        const size_t smem_r = (size_t)(maxM0 + nb) * 2 * sizeof(unsigned long long) + (size_t)maxM0 * 4;
        if (l2) hnsw_build_reverse_kernel<true><<<(unsigned)nt, HNSW_THREADS, smem_r, s>>>(g, n0, d_trip_sorted.p, nt);
        else hnsw_build_reverse_kernel<false><<<(unsigned)nt, HNSW_THREADS, smem_r, s>>>(g, n0, d_trip_sorted.p, nt);
        B200VS_CUDA(cudaGetLastError());
        phase(-1, s);
      }
      phases_finish(s);
      if (up_new > 0) B200VS_CUDA(cudaMemcpyAsync(up.data(), d_linkup.p, (size_t)up_new * 4, cudaMemcpyDeviceToHost, s));
      B200VS_CUDA(cudaMemcpyAsync(l0.data(), d_link0.p, l0.size() * 4, cudaMemcpyDeviceToHost, s));
      B200VS_CUDA(cudaStreamSynchronize(s));
    } catch (...) {
      // the mirror's link lists may hold part of the call: rebuild it from G, which is unchanged, at the next search
      for (auto& m : phase_marks) cudaEventDestroy(m.second);
      phase_marks.clear();
      dirty = true;
      uploaded_rows = 0;
      throw;
    }

    // ---- commit: G lays out the call's nodes and takes their rows in call order (add_point's bookkeeping), the device's link
    //      lists and the generator state ----
    G.append_nodes(lev);
    for (int64_t i = 0; i < n; ++i) G.take_label(in_ids[i], (tableint)(n0_call + i));
    memcpy(&G.data[(size_t)n0_call * dim], rows.data(), rows.size() * 4);
    memcpy(&G.labels[n0_call], in_ids, (size_t)n * 8);
    G.link0 = std::move(l0); G.linkup = std::move(up);
    G.n = ntot; G.enterpoint = ep; G.maxlevel = maxlevel; G.rng = rng;
    uploaded_rows = ntot;
    dirty = false;
  }

  // hnswlib getDataByLabel (hnsw.cc:383-395): the stored (for cosine: normalised) vector of a live label
  void reconstruct(int64_t n, const int64_t* in_ids, float* out, uint8_t* found) override {
    RwSharedGuard rl(this);
    for (int64_t i = 0; i < n; ++i) {
      auto it = G.lookup.find(in_ids[i]);
      const bool ok = it != G.lookup.end() && !G.deleted[it->second];
      if (found) found[i] = ok ? 1 : 0;
      if (ok) memcpy(out + (size_t)i * dim, G.vec(it->second), (size_t)dim * 4);
    }
  }
  // markDelete, hnsw.cc:256-281
  int64_t remove(int64_t n, const int64_t* del) override {
    std::unique_lock<std::shared_mutex> wl(rw);
    int64_t r = 0;
    for (int64_t i = 0; i < n; ++i) {
      auto it = G.lookup.find(del[i]);
      if (it == G.lookup.end()) continue;
      if (!G.deleted[it->second]) { G.deleted[it->second] = 1; ++G.ndeleted; ++r; }
    }
    if (r) dirty = true;
    return r;
  }

  std::mutex upload_mu;
  void upload(cudaStream_t s) {  // searches on different lanes may race to refresh the device mirror
    std::lock_guard<std::mutex> ul(upload_mu);
    if (!dirty) return;
    quiesce();  // earlier searches may still be reading the buffers this refresh reallocates
    const int64_t n = G.n;
    if (n == 0) { dirty = false; return; }
    d_data.reserve((size_t)std::max<int64_t>(n, (int64_t)(d_data.cap / dim)) * dim, (size_t)uploaded_rows * dim, s);
    if (n > uploaded_rows)
      B200VS_CUDA(cudaMemcpyAsync(d_data.p + (size_t)uploaded_rows * dim, G.data.data() + (size_t)uploaded_rows * dim,
                                  (size_t)(n - uploaded_rows) * dim * 4, cudaMemcpyHostToDevice, s));
    const size_t n0 = (size_t)n * (G.maxM0 + 1), pool = (size_t)G.up_off[n];
    d_labels.reserve(n, 0, s); d_link0.reserve(n0, 0, s); d_upoff.reserve(n + 1, 0, s); d_linkup.reserve(std::max<size_t>(pool, 1), 0, s);
    d_deleted.reserve(n, 0, s);
    B200VS_CUDA(cudaMemcpyAsync(d_labels.p, G.labels.data(), (size_t)n * 8, cudaMemcpyHostToDevice, s));
    B200VS_CUDA(cudaMemcpyAsync(d_link0.p, G.link0.data(), n0 * 4, cudaMemcpyHostToDevice, s));
    B200VS_CUDA(cudaMemcpyAsync(d_upoff.p, G.up_off.data(), (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, s));
    if (pool) B200VS_CUDA(cudaMemcpyAsync(d_linkup.p, G.linkup.data(), pool * 4, cudaMemcpyHostToDevice, s));
    B200VS_CUDA(cudaMemcpyAsync(d_deleted.p, G.deleted.data(), (size_t)n, cudaMemcpyHostToDevice, s));
    B200VS_CUDA(cudaStreamSynchronize(s));
    uploaded_rows = n;
    dirty = false;
  }

  // b200vs_search's efsearch refusal (hnsw.cc:332-336) and search's shared-memory refusal, from the arguments alone: a rank
  // whose graph is still empty returns from search before the latter, and a refused search must not leave its efsearch
  // in the sticky ef
  void check_row_search(int k, const b200vs_search_params* sp) const override {
    const int efs = sp ? sp->efsearch : 0;
    if (efs < 0 || efs > 1024)
      fail(B200VS_EILLEGAL_PARAMETERS, "efsearch is illegal, " + std::to_string(efs) + ", must between 0 and 1024");
    if (walk_smem_bytes(dim, std::max(efs > 0 ? efs : ef, k)) > HNSW_SMEM_LIMIT)
      fail(B200VS_EILLEGAL_PARAMETERS, "efsearch / dimension too large for the search kernel");
  }

  void search(const SearchReq& r, cudaStream_t s) override {
    refuse_probes(r);
    if (r.range) fail(B200VS_EVECTOR_NOT_SUPPORT, "range search not supported");
    if (r.raw) fail(B200VS_EVECTOR_NOT_SUPPORT, "raw-key search not supported");
    if (r.deep) fail(B200VS_EVECTOR_NOT_SUPPORT, "deep top-k is not implemented for HNSW");
    const SearchCtx& sc = *r.sc;
    const int64_t nq = r.nq;
    const int k = r.k;
    float* od = r.od;
    long long* oi = r.oi;
    if (sc.efsearch > 0) ef = sc.efsearch;  // sticky, mutated under the read lock like the reference (hnsw.cc:426-428)
    upload(s);
    if (G.n == 0) { fill_empty(r, s); return; }
    const float* q = queries(r, s);
    const int ef_run = std::max(ef, k);  // searchKnn: max(ef_, k)
    const HnswDev g = dev_graph(G.n, G.maxlevel, G.enterpoint, G.ndeleted > 0);
    const long long words = (G.n + 31) / 32;
    FilterDev f;
    f.has_range = sc.has_range; f.negate = sc.negate; f.rmin = sc.rmin; f.rmax = sc.rmax; f.sorted_ids = sc.sorted_ids_dev; f.n_ids = sc.n_ids;
    const size_t smem = walk_smem_bytes(dim, ef_run);
    if (smem > HNSW_SMEM_LIMIT) fail(B200VS_EILLEGAL_PARAMETERS, "efsearch / dimension too large for the search kernel");
    const bool fast = !(f.has_range || f.sorted_ids != nullptr) && !g.has_deletions && ef_run + 1 <= HNSW_CAND_SMEM && G.n < (1LL << 31);
    // the merged-array form keeps everything in shared memory; the heap form needs n + 1 candidate slots per query
    const long long cand_cap = fast ? 0 : G.n + 1;
    const int64_t chunk = fast ? nq : std::max<int64_t>(1, std::min<int64_t>(nq, (int64_t)(HNSW_CAND_POOL_BYTES / ((size_t)cand_cap * sizeof(HeapEnt)))));
    unsigned int* visited = scratch.alloc<unsigned int>((size_t)chunk * words);
    HeapEnt* cand = fast ? nullptr : scratch.alloc<HeapEnt>((size_t)chunk * cand_cap);
    ScopedKernelTimer timer(this, s, profiling);
    dispatch_walk(metric == B200VS_L2, fast, [&](auto L2_, auto FAST_) {
      const auto kernel = hnsw_search_kernel<decltype(L2_)::value, decltype(FAST_)::value>;
      B200VS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)HNSW_SMEM_LIMIT));
      for (int64_t a = 0; a < nq; a += chunk) {  // chunks share one visited / candidate pool, in stream order
        const int64_t m = std::min(chunk, nq - a);
        B200VS_CUDA(cudaMemsetAsync(visited, 0, (size_t)m * words * 4, s));
        kernel<<<(unsigned)m, HNSW_THREADS, smem, s>>>(g, q + (size_t)a * dim, m, k, ef_run, f, visited, words, cand, cand_cap,
                                                      od + (size_t)a * k, oi + (size_t)a * k);
        B200VS_CUDA(cudaGetLastError());
        launch_count(1);
      }
    });
    if (!fast) stats[6] += nq;
    timer.stop();
  }

  // the device mirror's rows, after upload(); a node's id is its label, or -1 once deleted.  The tile scan's row norms are
  // computed per call when asked for (the mirror keeps none).
  bool brute_force_rows(TcView& v, bool norms, cudaStream_t s) override {
    if (metric == B200VS_COSINE) fail(B200VS_EVECTOR_NOT_SUPPORT, "brute-force search of an HNSW cosine index is not supported");
    upload(s);
    if (G.n == 0) return false;
    const int64_t n = G.n;
    v.vecs = d_data.p;
    long long* ids = scratch.alloc<long long>(n);
    launch_node_ids(d_labels.p, d_deleted.p, n, ids, s);
    launch_count(1);
    v.ids = ids;
    if (norms) {
      float* nr = scratch.alloc<float>(n);
      launch_row_norms(d_data.p, n, dim, nr, s);
      launch_count(1);
      v.norms = nr;
      v.max_norm = device_max_norm(this, nr, n, s);
    }
    long long* off = scratch.alloc<long long>(1);
    int* len = scratch.alloc<int>(1);
    const int len1 = (int)std::min<int64_t>(n, 0x7fffffff);
    B200VS_CUDA(cudaMemsetAsync(off, 0, 8, s));
    B200VS_CUDA(cudaMemcpyAsync(len, &len1, 4, cudaMemcpyHostToDevice, s));
    set_flat_layout(v, n, off, len);
    return true;
  }

  int64_t count() const override { return G.n - G.ndeleted; }
  int64_t deleted_count() const override { return G.ndeleted; }
  // VectorIndexHnsw::NeedToRebuild, hnsw.cc:577-590: tombstones are more than half of every node, live or deleted
  bool need_rebuild() const override { return G.n > 0 && G.ndeleted > 0 && G.ndeleted > G.n / 2; }
  // the sources' live nodes with lo <= label <= hi, their stored rows (cosine: already normalised) in ascending label order,
  // gathered on the host (the rows live in the host graph), through the batched builder with the default batch; this fresh
  // index's level generator draws the levels, so the graph has no tombstones
  void live_ids(int64_t lo, int64_t hi, std::vector<int64_t>& out) override {
    for (int64_t i = 0; i < G.n; ++i)
      if (!G.deleted[i] && G.labels[i] >= lo && G.labels[i] <= hi) out.push_back(G.labels[i]);
  }
  int64_t rebuild_from(const std::vector<IndexBase*>& srcs, int64_t lo, int64_t hi) override {
    struct Live { int64_t label; const float* row; };
    std::vector<Live> live;
    for (IndexBase* src : srcs) {
      const HostGraph& S = static_cast<HnswIndex*>(src)->G;
      for (int64_t i = 0; i < S.n; ++i)
        if (!S.deleted[i] && S.labels[i] >= lo && S.labels[i] <= hi) live.push_back({S.labels[i], S.data.data() + (size_t)i * dim});
    }
    const int64_t n = (int64_t)live.size();
    if (n > max_element_limit) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from: dst max_elements is below the rows to copy");
    if (n == 0) return 0;
    std::sort(live.begin(), live.end(), [](const Live& a, const Live& b) { return a.label < b.label; });
    // the labels of one graph's live nodes are unique: a repeated label is held by two sources
    for (int64_t i = 1; i < n; ++i)
      if (live[i].label == live[i - 1].label)
        fail(B200VS_EVECTOR_ID_DUPLICATED, "rebuild_from_range: id " + std::to_string(live[i].label) + " is held by more than one source");
    std::vector<float> rows((size_t)n * dim);
    std::vector<int64_t> ids(n);
    for (int64_t i = 0; i < n; ++i) {
      ids[i] = live[i].label;
      memcpy(&rows[(size_t)i * dim], live[i].row, (size_t)dim * 4);
    }
    add_batched_locked(n, rows.data(), ids.data(), 0, true);
    return n;
  }
  int64_t memory_size() const override {
    return (int64_t)(G.n * ((G.maxM0 + 1) * 4 + (int64_t)dim * 4 + 8));  // hnsw.cc:612-623: per-element level-0 block
  }
  void export_lists(int64_t* list_off, float* vectors, uint8_t*, int64_t* out_ids) override {
    RwSharedGuard rl(this);
    int64_t o = 0;
    for (int64_t i = 0; i < G.n; ++i) {
      if (G.deleted[i]) continue;
      if (out_ids) out_ids[o] = G.labels[i];
      if (vectors) memcpy(vectors + (size_t)o * dim, G.vec((tableint)i), (size_t)dim * 4);
      ++o;
    }
    if (list_off) { list_off[0] = 0; list_off[1] = o; }
  }
  int64_t get_state(void* blob, size_t cap) override {
    RwSharedGuard rl(this);
    const int64_t n = G.n;
    const int64_t hdr[8] = {0x57534E48, n, dim, (int64_t)G.M, (int64_t)G.maxM0, G.maxlevel, (int64_t)G.enterpoint, (int64_t)metric};
    struct Section { const void* src; size_t bytes; bool pad8; };  // the blob's sections in order (DESIGN §5); pad8: zeros follow
    const Section secs[] = {{hdr, 64, false}, {G.levels.data(), (size_t)n * 4, true}, {G.up_off.data(), (size_t)(n + 1) * 8, false},
                            {G.link0.data(), (size_t)n * (G.maxM0 + 1) * 4, false}, {G.linkup.data(), (size_t)G.up_off[n] * 4, true},
                            {G.data.data(), (size_t)n * dim * 4, true}, {G.labels.data(), (size_t)n * 8, false},
                            {G.deleted.data(), G.ndeleted > 0 ? (size_t)n : 0, false}};  // tombstones only when anything is deleted
    auto end = [](size_t at, const Section& s) { return s.pad8 ? (at + s.bytes + 7) / 8 * 8 : at + s.bytes; };
    size_t sz = 0;
    for (const Section& s : secs) sz = end(sz, s);
    if (!blob || cap < sz) return (int64_t)sz;
    char* const base = (char*)blob;
    size_t at = 0;
    for (const Section& s : secs) {
      if (s.bytes) memcpy(base + at, s.src, s.bytes);
      memset(base + at + s.bytes, 0, end(at, s) - at - s.bytes);
      at = end(at, s);
    }
    return (int64_t)sz;
  }
};

IndexBase* make_hnsw(b200vs_metric m, int d, const b200vs_params& p) { return new HnswIndex(m, d, p); }

std::vector<int64_t> hnsw_state_labels(const IndexBase* ix, const void* blob, size_t len) {
  const HostGraph H = parse_state(static_cast<const HnswIndex*>(ix)->G, blob, len);
  std::vector<int64_t> live;
  for (int64_t i = 0; i < H.n; ++i) if (!H.deleted[i]) live.push_back(H.labels[i]);
  return live;
}

void hnsw_build_scratch_limit(IndexBase* ix, int64_t bytes) {
  std::unique_lock<std::shared_mutex> wl(ix->rw);
  static_cast<HnswIndex*>(ix)->build_scratch_limit = bytes;
}

}  // namespace b200vs
