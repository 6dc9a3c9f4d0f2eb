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
// Search kernel (hnsw_search_kernel): one warp per query.  Upper layers: greedy descent.  Base layer: the
// reference's searchBaseLayerST loop — pop the closest candidate, gather its <= 2M neighbour rows, compute the
// unvisited neighbours' distances as one batch (8 quads per warp, exact AVX-512 order, so the traversal is
// identical to the CPU traversal), then apply the heap updates in neighbour order.
#include <algorithm>
#include <cmath>
#include <queue>
#include <memory>
#include <mutex>
#include <random>
#include <thread>

#include "index.h"
#include "scan_kernels.cuh"

namespace b200vs {

void fill_empty_results(int64_t nq, int k, float* od, long long* oi, cudaStream_t s);

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

struct HostGraph {
  int metric, d;
  size_t M, maxM, maxM0, efc;
  double mult;
  std::default_random_engine rng;
  int64_t n = 0, cap = 0;
  int maxlevel = -1;
  tableint enterpoint = (tableint)-1;
  std::vector<float> data;
  std::vector<int64_t> labels;
  std::vector<int> levels;
  std::vector<tableint> link0;
  std::vector<std::vector<tableint>> linkup;
  std::vector<uint8_t> deleted;
  std::unordered_map<int64_t, tableint> lookup;
  std::vector<uint32_t> visited;
  uint32_t tag = 0;
  int64_t ndeleted = 0;
  // concurrent insertion (hnswlib's locking scheme): one lock per node for its link lists, one for the entry point /
  // max level, one for slot allocation + label map + level generator; every worker owns a visited-tag array
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
  void reserve(int64_t ncap) {  // resizeIndex
    if (ncap <= cap) return;
    data.resize((size_t)ncap * d); labels.resize(ncap); levels.resize(ncap); link0.resize((size_t)ncap * (maxM0 + 1), 0);
    linkup.resize(ncap); deleted.resize(ncap, 0); visited.resize(ncap, 0);
    cap = ncap;
  }
  const float* vec(tableint i) const { return &data[(size_t)i * d]; }
  float dist(const float* a, const float* b) const {
    if (metric == B200VS_L2) return host_avx512_order<true>(a, b, d);
    return 1.0f - host_avx512_order<false>(a, b, d);
  }
  tableint* ll(tableint i, int level) { return level == 0 ? &link0[(size_t)i * (maxM0 + 1)] : &linkup[i][(size_t)(level - 1) * (maxM + 1)]; }

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
  // insert at once (the reference's ParallelFor over addPoint, vector_index_hnsw.cc:229-243); capacity and locks are
  // reserved by the caller, so no container is re-allocated while workers run.
  template <bool MT>
  void add_point(const float* x, int64_t label, VisitCtx* vc = nullptr) {
    tableint cur_c;
    int curlevel;
    {
      std::unique_lock<std::mutex> al;
      if (MT) al = std::unique_lock<std::mutex>(lk->alloc_mu);
      auto it = lookup.find(label);
      if (it != lookup.end()) { if (!deleted[it->second]) { deleted[it->second] = 1; ++ndeleted; } lookup.erase(it); }
      if (!MT && n >= cap) reserve(std::max<int64_t>(1024, cap * 2));
      cur_c = (tableint)n++;
      lookup[label] = cur_c;
      std::uniform_real_distribution<double> U(0.0, 1.0);
      curlevel = (int)(-log(U(rng)) * mult);
    }
    std::unique_lock<std::mutex> own;
    if (MT) own = std::unique_lock<std::mutex>(node_mu[cur_c]);
    std::unique_lock<std::mutex> gl;
    if (MT) gl = std::unique_lock<std::mutex>(lk->global_mu);
    const int maxlevelcopy = maxlevel;
    if (MT && curlevel <= maxlevelcopy) gl.unlock();
    tableint cur = enterpoint;
    memcpy(&data[(size_t)cur_c * d], x, sizeof(float) * d);
    labels[cur_c] = label; levels[cur_c] = curlevel; deleted[cur_c] = 0;
    memset(&link0[(size_t)cur_c * (maxM0 + 1)], 0, (maxM0 + 1) * sizeof(tableint));
    linkup[cur_c].assign((size_t)curlevel * (maxM + 1), 0);
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

// ---------------- device search ----------------
struct HnswDev {
  const float* data;
  const long long* labels;
  const unsigned int* link0;
  const long long* up_off;
  const unsigned int* linkup;
  const unsigned char* deleted;
  long long n;
  int d, maxM, maxM0, maxlevel, l2;
  unsigned int enterpoint;
  int has_deletions;
};

constexpr int HNSW_THREADS = 128;   // one CTA per query: warp 0 walks the graph, all 32 quads score a hop's neighbours together
constexpr int HNSW_CAND_SMEM = 1024; // candidate-heap entries kept in shared memory (the levels near the root); deeper ones spill to global
// Heap form: the visited set admits every node to the candidate heap at most once, so n + 1 entries per query always
// suffice.  When nq · (n + 1) entries exceed this budget the queries run in chunks of fewer CTAs.
constexpr size_t HNSW_CAND_POOL_BYTES = 512ull << 20;

struct HeapEnt { float d; unsigned int id; };

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

// One CTA (128 threads) per query.  Warp 0 runs hnswlib's control flow (greedy descent of the upper layers, then
// searchBaseLayerST): it pops the closest candidate, reads its link list 32 neighbours at a time, keeps the unvisited ones in
// list order; then ALL 32 quads of the CTA compute those rows' distances in one round (exact AVX-512 order, so the traversal
// is the CPU traversal); lane 0 applies the heap updates in neighbour order.  Two block barriers per batch of <= 32 neighbours.
// FAST (no id filter, no tombstones — every accepted neighbour enters both of hnswlib's queues): the two binary heaps collapse
// into ONE ascending array T of the best <= ef nodes with an "expanded" flag per entry.  The next candidate is the first
// unexpanded entry of T; a hop's <= 32 scored neighbours are merged into T by all 128 threads at once (each thread places one
// old entry and at most one new one at its rank), instead of ~30 sift-up / sift-down sequences executed by a single lane at one
// dependent instruction per ~25 ns — that lone-lane heap work was 80 % of a hop.  The visited set, the order in which nodes
// are expanded and the returned ids / distances are those of searchBaseLayerST (exact-distance ties between different nodes,
// which std::priority_queue orders by heap position, are the one place the two can differ).
template <bool L2, bool FAST>
__global__ void __launch_bounds__(HNSW_THREADS) hnsw_search_kernel(const HnswDev g, const float* __restrict__ queries, long long nq,
                                                                  int k, int ef, FilterDev filt, unsigned int* visited /*[nq, words]*/,
                                                                  long long words, HeapEnt* cand_pool, long long cand_cap, float* out_dist,
                                                                  long long* out_ids) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ float s_d[32];
  __shared__ unsigned int s_id[32];
  __shared__ int s_m;  // rows to score this round; -1 = the walk is over
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long qi = blockIdx.x;
  const int d = g.d;
  const size_t qbytes = ((size_t)d * 4 + 15) / 16 * 16;
  float* qs = reinterpret_cast<float*>(smem);
  HeapEnt* top_sm = reinterpret_cast<HeapEnt*>(smem + qbytes);                                   // [ef + 1]
  HeapEnt* cand_sm = reinterpret_cast<HeapEnt*>(smem + qbytes + (size_t)(ef + 1) * sizeof(HeapEnt));  // [HNSW_CAND_SMEM]
  for (int i = threadIdx.x; i < d; i += HNSW_THREADS) qs[i] = queries[(size_t)qi * d + i];
  if (g.n == 0) {
    for (int i = threadIdx.x; i < k; i += HNSW_THREADS) { out_dist[(size_t)qi * k + i] = 0.f; out_ids[(size_t)qi * k + i] = -1; }
    return;
  }
  __syncthreads();
  const bool vec = (d & 3) == 0;
  const int quad = threadIdx.x >> 2, t = threadIdx.x & 3;
  unsigned int* vis = visited + (size_t)qi * words;
  const HeapRef top{top_sm, top_sm, ef + 1};
  const HeapRef cand{cand_sm, cand_pool + (size_t)qi * cand_cap, HNSW_CAND_SMEM};
  const bool filtered = filt.has_range || filt.sorted_ids != nullptr;
  const bool strict_stop = filtered || g.has_deletions;

  // distances of s_id[0..m) -> s_d[0..m): one row per quad, every thread of the CTA calls (m <= 32)
  auto score = [&](int m) {
    const unsigned int row = s_id[quad < m ? quad : 0];
    float v = quad_distance<L2>(g.data + (size_t)row * d, qs, d, t, vec);
    if (!L2) v = __fsub_rn(1.0f, v);  // hnswlib InnerProductDistance
    if (quad < m && t == 0) s_d[quad] = v;
  };

  // ---- entry point ----
  unsigned int cur = g.enterpoint;
  if (threadIdx.x == 0) s_id[0] = cur;
  __syncthreads();
  score(1);
  __syncthreads();
  float curdist = s_d[0];
  // ---- upper layers: greedy descent (every thread tracks the same state) ----
  for (int level = g.maxlevel; level > 0; --level) {
    bool changed = true;
    while (changed) {
      changed = false;
      const unsigned int* l = g.linkup + g.up_off[cur] + (size_t)(level - 1) * (g.maxM + 1);
      const int size = (int)l[0];
      for (int c0 = 0; c0 < size; c0 += 32) {
        const int m = min(32, size - c0);
        __syncthreads();  // previous round's s_d / s_id fully consumed
        if (warp == 0 && lane < m) s_id[lane] = l[1 + c0 + lane];
        __syncthreads();
        score(m);
        __syncthreads();
        for (int i = 0; i < m; ++i) {
          const float dd = s_d[i];
          if (dd < curdist) { curdist = dd; cur = s_id[i]; changed = true; }
        }
      }
    }
  }
  if (FAST) {
    // ---- base layer, merged-array form.  T = cand_sm region reused: [2][ef] entries (id bit 31 = expanded) ----
    HeapEnt* T = top_sm;            // [ef + 1]
    HeapEnt* T2 = cand_sm;          // [>= ef + 1] (HNSW_CAND_SMEM >= ef + 1 is checked on the host)
    int ntop = 1;
    if (threadIdx.x == 0) { T[0].d = curdist; T[0].id = cur; vis[cur >> 5] |= 1u << (cur & 31); }
    unsigned int node = 0;
    int size = 0, c0 = 0;
    bool expanding = false;
    for (;;) {
      __syncthreads();  // (A) T complete, s_d / s_id of the previous round consumed
      if (warp == 0) {
        int m = -1;
        for (;;) {
          if (!expanding) {
            int idx = -1;
            for (int b0 = 0; b0 < ntop && idx < 0; b0 += 32) {  // first unexpanded entry = closest open candidate
              const int i = b0 + lane;
              const bool open = i < ntop && (T[i].id >> 31) == 0u;
              const unsigned msk = __ballot_sync(0xffffffffu, open);
              if (msk) idx = b0 + __ffs(msk) - 1;
            }
            if (idx < 0) { m = -1; break; }
            node = T[idx].id;
            __syncwarp();
            if (lane == 0) T[idx].id = node | 0x80000000u;
            size = (int)g.link0[(size_t)node * (g.maxM0 + 1)];
            c0 = 0;
            expanding = true;
          }
          if (c0 >= size) { expanding = false; continue; }
          const unsigned int* l = g.link0 + (size_t)node * (g.maxM0 + 1) + 1 + c0;
          const int cnt = min(32, size - c0);
          c0 += 32;
          unsigned int nb = 0;
          bool fresh = false;
          if (lane < cnt) { nb = l[lane]; fresh = ((vis[nb >> 5] >> (nb & 31)) & 1u) == 0u; }
          const unsigned int mask = __ballot_sync(0xffffffffu, fresh);
          if (fresh) {
            atomicOr(&vis[nb >> 5], 1u << (nb & 31));
            s_id[__popc(mask & ((1u << lane) - 1u))] = nb;
          }
          m = __popc(mask);
          if (m > 0) break;
        }
        if (lane == 0) s_m = m;
      }
      __syncthreads();  // (B)
      const int m = s_m;
      if (m < 0) break;
      score(m);
      __syncthreads();  // (C) s_d complete
      // merge the m scored neighbours into T (ascending, old entries first among equals), keep the best ef
      for (int tix = threadIdx.x; tix < ntop; tix += HNSW_THREADS) {
        const HeapEnt e = T[tix];
        int c = 0;
        for (int j = 0; j < m; ++j) c += s_d[j] < e.d ? 1 : 0;
        if (tix + c < ef) T2[tix + c] = e;
      }
      if (threadIdx.x < m) {
        const float dj = s_d[threadIdx.x];
        int rank = 0;
        for (int i = 0; i < m; ++i) rank += (s_d[i] < dj || (s_d[i] == dj && i < (int)threadIdx.x)) ? 1 : 0;
        int lo = 0, hi = ntop;  // number of old entries with d <= dj
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (T[mid].d <= dj) lo = mid + 1; else hi = mid; }
        if (rank + lo < ef) { HeapEnt e; e.d = dj; e.id = s_id[threadIdx.x]; T2[rank + lo] = e; }
      }
      ntop = min(ef, ntop + m);
      HeapEnt* tmp = T; T = T2; T2 = tmp;
    }
    __syncthreads();
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
  // ---- base layer: searchBaseLayerST ----
  int ntop = 0, ncand = 0;
  float lower = 3.402823466e+38f;
  if (warp == 0) {
    const long long lab = g.labels[cur];
    const bool ok = !g.deleted[cur] && filter_pass(filt, lab);
    if (lane == 0) {
      if (ok) { h_push<true>(top, ntop, curdist, cur); h_push<false>(cand, ncand, curdist, cur); }
      else h_push<false>(cand, ncand, 3.402823466e+38f, cur);
      vis[cur >> 5] |= 1u << (cur & 31);
    }
    lower = ok ? curdist : 3.402823466e+38f;
  }
  // warp 0 state that survives across rounds: the node being expanded and how far into its link list we are
  unsigned int node = 0;
  int size = 0, c0 = 0;
  bool expanding = false;
  for (;;) {
    __syncthreads();  // (A) s_d / s_id of the previous round consumed by everyone
    if (warp == 0) {
      int m = -1;
      for (;;) {  // find the next non-empty batch of unvisited neighbours
        if (!expanding) {
          int go = 0;
          if (lane == 0 && ncand > 0) {
            const HeapEnt ce = cand.get(0);
            const bool stop = ce.d > lower && (ntop == ef || !strict_stop);
            if (!stop) { node = ce.id; h_pop<false>(cand, ncand); go = 1; }
          }
          go = __shfl_sync(0xffffffffu, go, 0);
          if (!go) { m = -1; break; }
          node = __shfl_sync(0xffffffffu, node, 0);
          size = (int)g.link0[(size_t)node * (g.maxM0 + 1)];
          c0 = 0;
          expanding = true;
        }
        if (c0 >= size) { expanding = false; continue; }
        const unsigned int* l = g.link0 + (size_t)node * (g.maxM0 + 1) + 1 + c0;
        const int cnt = min(32, size - c0);
        c0 += 32;
        unsigned int nb = 0;
        bool fresh = false;
        if (lane < cnt) { nb = l[lane]; fresh = ((vis[nb >> 5] >> (nb & 31)) & 1u) == 0u; }
        const unsigned int mask = __ballot_sync(0xffffffffu, fresh);
        if (fresh) {
          atomicOr(&vis[nb >> 5], 1u << (nb & 31));
          s_id[__popc(mask & ((1u << lane) - 1u))] = nb;
        }
        m = __popc(mask);
        if (m > 0) break;
      }
      if (lane == 0) s_m = m;
    }
    __syncthreads();  // (B) s_id / s_m published
    const int m = s_m;
    if (m < 0) break;
    score(m);
    __syncthreads();  // (C) s_d complete
    if (warp == 0) {
      bool allowed = false;
      if (lane < m) { const unsigned int c = s_id[lane]; allowed = !g.deleted[c] && filter_pass(filt, g.labels[c]); }
      const unsigned int amask = __ballot_sync(0xffffffffu, allowed);
      if (lane == 0) {
        for (int i = 0; i < m; ++i) {
          const float dd = s_d[i];
          if (ntop < ef || lower > dd) {
            h_push<false>(cand, ncand, dd, s_id[i]);  // fresh nodes only: ncand <= n < cand_cap
            if ((amask >> i) & 1u) h_push<true>(top, ntop, dd, s_id[i]);
            if (ntop > ef) h_pop<true>(top, ntop);
            if (ntop > 0) lower = top.get(0).d;
          }
        }
      }
      lower = __shfl_sync(0xffffffffu, lower, 0);
    }
  }
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

}  // namespace

struct HnswIndex : IndexBase {
  HostGraph G;
  int64_t max_element_limit;
  int ef = 10;  // hnswlib default; sticky setEf (hnsw.cc:426-428)
  bool dirty = true;
  int64_t uploaded_rows = 0;
  DevBuf<float> d_data;
  DevBuf<long long> d_labels, d_upoff;
  DevBuf<unsigned int> d_link0, d_linkup;
  DevBuf<unsigned char> d_deleted;

  HnswIndex(b200vs_metric m, int d, const b200vs_params& p) : IndexBase(B200VS_HNSW, m, d, p) {
    if (p.hnsw_m <= 0 || p.hnsw_efc <= 0) fail(B200VS_EILLEGAL_PARAMETERS, "hnsw nlinks / efconstruction must be > 0");
    max_element_limit = p.max_elements > 0 ? p.max_elements : (1LL << 40);
    G.init(metric, d, p.hnsw_m, p.hnsw_efc, 100);  // random_seed = 100, hnsw.cc:181-182
  }

  // blob (the oracle's / this index's export): int64 hdr[8] = {'HNSW', n, d, M, maxM0, maxlevel, enterpoint, metric};
  // int32 levels[n]; (pad 8) int64 up_off[n+1]; uint32 link0[n*(maxM0+1)]; uint32 linkup[up_off[n]]; (pad 8)
  // float data[n*d]; (pad 8) int64 labels[n]
  void set_state(const void* blob, size_t len) override {
    std::unique_lock<std::shared_mutex> wl(rw);
    if (len < 64) fail(B200VS_EILLEGAL_PARAMETERS, "state blob too short");
    const char* base = (const char*)blob;
    const int64_t* hdr = (const int64_t*)base;
    if (hdr[0] != 0x57534E48 || hdr[2] != dim || hdr[3] != (int64_t)G.M) fail(B200VS_EILLEGAL_PARAMETERS, "bad HNSW state blob");
    const int64_t n = hdr[1];
    {  // the blob must hold every section BEFORE anything is copied out of it
      if (n < 0 || n > (1LL << 31)) fail(B200VS_EILLEGAL_PARAMETERS, "bad HNSW state blob (row count)");
      auto pad8 = [](uint64_t v) { return (v + 7) / 8 * 8; };
      uint64_t need = pad8(64 + (uint64_t)n * 4) + (uint64_t)(n + 1) * 8;
      if (len < need) fail(B200VS_EILLEGAL_PARAMETERS, "state blob truncated");
      const int64_t* off_chk = (const int64_t*)((const char*)blob + pad8(64 + (uint64_t)n * 4));
      const int64_t up = off_chk[n];
      if (up < 0 || up > (int64_t)(len / 4)) fail(B200VS_EILLEGAL_PARAMETERS, "bad HNSW state blob (link pool)");
      need = pad8(need + (uint64_t)n * (2 * G.M + 1) * 4 + (uint64_t)up * 4);
      need = pad8(need + (uint64_t)n * dim * 4) + (uint64_t)n * 8;
      if (len < need) fail(B200VS_EILLEGAL_PARAMETERS, "state blob truncated");
    }
    HostGraph H;
    H.init(metric, dim, (int)G.M, (int)G.efc, 100);
    H.reserve(std::max<int64_t>(n, 1));
    const char* p = base + 64;
    memcpy(H.levels.data(), p, n * 4); p += n * 4;
    p = base + ((p - base) + 7) / 8 * 8;
    const int64_t* off = (const int64_t*)p; p += (n + 1) * 8;
    memcpy(H.link0.data(), p, (size_t)n * (H.maxM0 + 1) * 4); p += (size_t)n * (H.maxM0 + 1) * 4;
    for (int64_t i = 0; i < n; ++i) { H.linkup[i].assign((const tableint*)p + off[i], (const tableint*)p + off[i + 1]); }
    p += off[n] * 4;
    p = base + ((p - base) + 7) / 8 * 8;
    memcpy(H.data.data(), p, (size_t)n * dim * 4); p += (size_t)n * dim * 4;
    p = base + ((p - base) + 7) / 8 * 8;
    memcpy(H.labels.data(), p, n * 8);
    if ((size_t)(p - base) + (size_t)n * 8 > len) fail(B200VS_EILLEGAL_PARAMETERS, "state blob truncated");
    H.n = n; H.maxlevel = (int)hdr[5]; H.enterpoint = (tableint)hdr[6];
    const size_t after_labels = (size_t)(p - base) + (size_t)n * 8;
    if (len >= after_labels + (size_t)n) {  // optional trailing tombstone bytes (written only when something was deleted)
      memcpy(H.deleted.data(), base + after_labels, (size_t)n);
      for (int64_t i = 0; i < n; ++i) H.ndeleted += H.deleted[i] ? 1 : 0;
    }
    for (int64_t i = 0; i < n; ++i) if (!H.deleted[i]) H.lookup[H.labels[i]] = (tableint)i;
    G = std::move(H);
    dirty = true; uploaded_rows = 0;
  }

  // VectorIndexHnsw::Upsert, hnsw.cc:203-254 (Add == Upsert; vectors are normalised per row for cosine)
  void add(int64_t n, const float* x, const int64_t* in_ids, bool) override {
    std::unique_lock<std::shared_mutex> wl(rw);
    if (G.n + n > max_element_limit) fail(B200VS_EINTERNAL, "upsert failed, exceeds max elements");
    auto prepared = [&](int64_t i, std::vector<float>& tmp) -> const float* {
      const float* xi = x + (size_t)i * dim;
      if (metric != B200VS_COSINE) return xi;
      float norm = 0.0f;  // NormalizeVectorForHnsw, vector_index_utils.cc:493-500
      for (int j = 0; j < dim; ++j) norm += xi[j] * xi[j];
      norm = 1.0f / (sqrtf(norm) + 1e-30f);
      for (int j = 0; j < dim; ++j) tmp[j] = xi[j] * norm;
      return tmp.data();
    };
    const int nthreads = (int)std::min<int64_t>(std::max(1, params.hnsw_build_threads), n);
    if (nthreads <= 1) {  // single writer: deterministic graph (equal to the oracle's for the same insertion order)
      std::vector<float> tmp(dim);
      for (int64_t i = 0; i < n; ++i) G.add_point<false>(prepared(i, tmp), in_ids[i]);
    } else {  // concurrent insertion, as the reference's thread pool does (hnsw.cc:229-243)
      G.reserve(std::max<int64_t>(G.cap, G.n + n));
      G.reserve_locks(G.cap);
      std::atomic<int64_t> next{0};
      if (G.n == 0) { std::vector<float> tmp(dim); G.add_point<false>(prepared(0, tmp), in_ids[0]); next = 1; }  // hnswlib: first element alone
      std::vector<std::thread> ts;
      for (int t = 0; t < nthreads; ++t)
        ts.emplace_back([&]() {
          HostGraph::VisitCtx vc;
          vc.visited.assign((size_t)G.cap, 0u);
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
    d_labels.reserve(n, 0, s); d_link0.reserve((size_t)n * (G.maxM0 + 1), 0, s); d_upoff.reserve(n + 1, 0, s); d_deleted.reserve(n, 0, s);
    std::vector<long long> off(n + 1);
    long long acc = 0;
    for (int64_t i = 0; i < n; ++i) { off[i] = acc; acc += (long long)G.linkup[i].size(); }
    off[n] = acc;
    std::vector<unsigned int> up((size_t)std::max<long long>(acc, 1));
    for (int64_t i = 0; i < n; ++i) if (!G.linkup[i].empty()) memcpy(&up[off[i]], G.linkup[i].data(), G.linkup[i].size() * 4);
    d_linkup.reserve(up.size(), 0, s);
    B200VS_CUDA(cudaMemcpyAsync(d_labels.p, G.labels.data(), (size_t)n * 8, cudaMemcpyHostToDevice, s));
    B200VS_CUDA(cudaMemcpyAsync(d_link0.p, G.link0.data(), (size_t)n * (G.maxM0 + 1) * 4, cudaMemcpyHostToDevice, s));
    B200VS_CUDA(cudaMemcpyAsync(d_upoff.p, off.data(), (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, s));
    B200VS_CUDA(cudaMemcpyAsync(d_linkup.p, up.data(), up.size() * 4, cudaMemcpyHostToDevice, s));
    B200VS_CUDA(cudaMemcpyAsync(d_deleted.p, G.deleted.data(), (size_t)n, cudaMemcpyHostToDevice, s));
    B200VS_CUDA(cudaStreamSynchronize(s));
    uploaded_rows = n;
    dirty = false;
  }

  void search_dev(int64_t nq, const float* xq, int k, const SearchCtx& sc, float* od, long long* oi, cudaStream_t s) override {
    if (sc.efsearch > 0) ef = sc.efsearch;  // sticky, mutated under the read lock like the reference (hnsw.cc:426-428)
    upload(s);
    if (G.n == 0) { fill_empty_results(nq, k, od, oi, s); return; }
    const float* q = prepare_queries(nq, xq, s);
    const int ef_run = std::max(ef, k);  // searchKnn: max(ef_, k)
    HnswDev g;
    g.data = d_data.p; g.labels = d_labels.p; g.link0 = d_link0.p; g.up_off = d_upoff.p; g.linkup = d_linkup.p; g.deleted = d_deleted.p;
    g.n = G.n; g.d = dim; g.maxM = (int)G.maxM; g.maxM0 = (int)G.maxM0; g.maxlevel = G.maxlevel; g.l2 = metric == B200VS_L2;
    g.enterpoint = G.enterpoint; g.has_deletions = G.ndeleted > 0;
    const long long words = (G.n + 31) / 32;
    FilterDev f;
    f.has_range = sc.has_range; f.negate = sc.negate; f.rmin = sc.rmin; f.rmax = sc.rmax; f.sorted_ids = sc.sorted_ids_dev; f.n_ids = sc.n_ids;
    const size_t qbytes = ((size_t)dim * 4 + 15) / 16 * 16;
    const size_t smem = qbytes + (size_t)(ef_run + 1) * sizeof(HeapEnt) + (size_t)HNSW_CAND_SMEM * sizeof(HeapEnt);
    if (smem > 200 * 1024) fail(B200VS_EILLEGAL_PARAMETERS, "efsearch / dimension too large for the search kernel");
    const bool fast = !(f.has_range || f.sorted_ids != nullptr) && !g.has_deletions && ef_run + 1 <= HNSW_CAND_SMEM && G.n < (1LL << 31);
    // the merged-array form keeps everything in shared memory; the heap form needs n + 1 candidate slots per query
    const long long cand_cap = fast ? 0 : G.n + 1;
    const int64_t chunk = fast ? nq : std::max<int64_t>(1, std::min<int64_t>(nq, (int64_t)(HNSW_CAND_POOL_BYTES / ((size_t)cand_cap * sizeof(HeapEnt)))));
    unsigned int* visited = scratch.alloc<unsigned int>((size_t)chunk * words);
    HeapEnt* cand = fast ? nullptr : scratch.alloc<HeapEnt>((size_t)chunk * cand_cap);
    ScopedKernelTimer timer(this, s, profiling);
#define B200VS_HNSW_LAUNCH(L2_, FAST_)                                                                                              \
  do {                                                                                                                             \
    B200VS_CUDA(cudaFuncSetAttribute(hnsw_search_kernel<L2_, FAST_>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));     \
    hnsw_search_kernel<L2_, FAST_><<<(unsigned)m, HNSW_THREADS, smem, s>>>(g, q + (size_t)a * dim, m, k, ef_run, f, visited, words,  \
                                                                          cand, cand_cap, od + (size_t)a * k, oi + (size_t)a * k);  \
  } while (0)
    for (int64_t a = 0; a < nq; a += chunk) {  // chunks share one visited / candidate pool, in stream order
      const int64_t m = std::min(chunk, nq - a);
      B200VS_CUDA(cudaMemsetAsync(visited, 0, (size_t)m * words * 4, s));
      if (g.l2) { if (fast) B200VS_HNSW_LAUNCH(true, true); else B200VS_HNSW_LAUNCH(true, false); }
      else { if (fast) B200VS_HNSW_LAUNCH(false, true); else B200VS_HNSW_LAUNCH(false, false); }
      B200VS_CUDA(cudaGetLastError());
      launch_count(1);
    }
#undef B200VS_HNSW_LAUNCH
    if (!fast) stats[6] += nq;
    timer.stop();
  }

  int64_t count() const override { return G.n - G.ndeleted; }
  int64_t deleted_count() const override { return G.ndeleted; }
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
    int64_t up = 0;
    for (int64_t i = 0; i < n; ++i) up += (int64_t)G.linkup[i].size();
    auto pad8 = [](int64_t v) { return (v + 7) / 8 * 8; };
    int64_t sz = pad8(64 + n * 4);
    sz = pad8(sz + (n + 1) * 8 + n * (int64_t)(G.maxM0 + 1) * 4 + up * 4);
    sz = pad8(sz + n * (int64_t)dim * 4);
    sz += n * 8;
    if (G.ndeleted > 0) sz += n;  // trailing tombstone bytes
    if (!blob || (int64_t)cap < sz) return sz;
    char* base = (char*)blob;
    char* p = base;
    int64_t hdr[8] = {0x57534E48, n, dim, (int64_t)G.M, (int64_t)G.maxM0, G.maxlevel, (int64_t)G.enterpoint, (int64_t)metric};
    memcpy(p, hdr, 64); p += 64;
    memcpy(p, G.levels.data(), n * 4); p += n * 4;
    p = base + pad8(p - base);
    int64_t* off = (int64_t*)p; p += (n + 1) * 8;
    int64_t acc = 0;
    for (int64_t i = 0; i < n; ++i) { off[i] = acc; acc += (int64_t)G.linkup[i].size(); }
    off[n] = acc;
    memcpy(p, G.link0.data(), (size_t)n * (G.maxM0 + 1) * 4); p += (size_t)n * (G.maxM0 + 1) * 4;
    for (int64_t i = 0; i < n; ++i) { memcpy(p, G.linkup[i].data(), G.linkup[i].size() * 4); p += G.linkup[i].size() * 4; }
    p = base + pad8(p - base);
    memcpy(p, G.data.data(), (size_t)n * dim * 4); p += (size_t)n * dim * 4;
    p = base + pad8(p - base);
    memcpy(p, G.labels.data(), n * 8); p += n * 8;
    if (G.ndeleted > 0) memcpy(p, G.deleted.data(), (size_t)n);
    return sz;
  }
};

IndexBase* make_hnsw(b200vs_metric m, int d, const b200vs_params& p) { return new HnswIndex(m, d, p); }

}  // namespace b200vs
