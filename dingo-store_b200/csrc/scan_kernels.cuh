// scan_kernels.cuh — exact FP32 scan + select kernels (the engine's always-correct path).
//
// These kernels replace, bit-for-bit in the reference's AVX-512 evaluation order, the CPU loops that
// dingo-store reaches through faiss:
//   exhaustive_{L2sqr,inner_product}_seq  <- IndexFlat::search   <- VectorIndexFlat::Search   (vector_index_flat.cc:249-252)
//   IVFFlatScanner::scan_codes            <- IndexIVFFlat::search <- VectorIndexIvfFlat::Search (vector_index_ivf_flat.cc:247-251)
//   the IndexFlat coarse quantiser of IVF (vector_index_ivf_flat.cc:805-837) and add-time assignment.
// They are also the rerank stage of the tensor-core candidate pass (tc_ivf.cuh) and its fallback.
#pragma once
#include "common.cuh"
#include "deep_select.cuh"
#include "filter.cuh"
#include "select.cuh"

namespace b200vs {

struct ScanArgs {
  const float* vecs;        // [rows, d]
  const long long* ids;     // [rows], <0 = removed slot
  const float* queries;     // [nq, d] (already normalised for cosine)
  int d;
  int mode;                 // 0: one segment [0,n)   1: IVF probes
  long long n;              // mode 0
  const long long* probes;  // mode 1: [nq, nprobe] list indices (may contain -1)
  int nprobe;
  const long long* list_off;  // [nlist]
  const int* list_len;        // [nlist]
  int k;
  int nsplit;
  uint32_t* ws_kd;     // [nq, nsplit, k]
  long long* ws_kid;   // [nq, nsplit, k]
  FilterDev filt;
  int has_thr;         // range search: fixed initial threshold key
  uint32_t thr_key;
  int pool_cap;
  const int* qmap;    // optional: blockIdx.y -> query index (exact re-run of uncertified queries)
  const int* qcount;  // optional: number of live entries in qmap (blocks beyond it exit)
};

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_QUADS = SCAN_THREADS / 4;

inline size_t scan_smem_bytes(int d, int nprobe, int pool_cap) {
  size_t q = ((size_t)d * 4 + 15) / 16 * 16;
  size_t pf = ((size_t)(nprobe + 1) * 4 + 15) / 16 * 16;
  return q + pf + BlockSelect::smem_bytes(pool_cap);
}

// Per-row distance of the exact scan.  Fp32Dist: the reference's FP32 order (quad_distance); d = floats per row.
template <bool L2>
struct Fp32Dist {
  static constexpr bool kL2 = L2;
  static __device__ __forceinline__ float eval(const float* vecs, long long row, const float* qs, int d, int t, bool vec) {
    return quad_distance<L2>(vecs + (size_t)row * d, qs, d, t, vec);
  }
};
// HammingDist: binary rows, d = 32-bit words per (zero-padded) row, vecs / qs hold the words.  sum popc(q ^ x) over the
// row in int, returned as float: exact (<= 32768 bits), so the key f2ord(dist) orders rows like the integer distance.
// Thread t of the quad takes words 4t..4t+3 of every 16-word chunk (vec: 16-byte loads) or words t, t+4, ...
struct HammingDist {
  static constexpr bool kL2 = true;
  static __device__ __forceinline__ float eval(const float* vecs, long long row, const float* qs, int d, int t, bool vec) {
    const uint32_t* x = reinterpret_cast<const uint32_t*>(vecs) + (size_t)row * d;
    const uint32_t* q = reinterpret_cast<const uint32_t*>(qs);
    int s = 0;
    if (vec) {
      for (int i = 4 * t; i < d; i += 16) {
        const uint4 a = *reinterpret_cast<const uint4*>(x + i), b = *reinterpret_cast<const uint4*>(q + i);
        s += __popc(a.x ^ b.x) + __popc(a.y ^ b.y) + __popc(a.z ^ b.z) + __popc(a.w ^ b.w);
      }
    } else {
      for (int i = t; i < d; i += 4) s += __popc(x[i] ^ q[i]);
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1, 4);
    s += __shfl_xor_sync(0xffffffffu, s, 2, 4);
    return (float)s;
  }
};

// The exact scan of one query's candidates [r0, r1) of split `split`: every eligible row (a live id that passes the filters)
// goes to the sink with its key and candidate-space position.  Sink: SelectSink (top-k) or DeepKeySink (deep top-k).
template <class Dist, class Sink>
static __device__ __forceinline__ void scan_rows(const ScanArgs& a, unsigned char* smem, const int split, const int qi, Sink& sink) {
  const int d = a.d;
  float* qs = reinterpret_cast<float*>(smem);
  const size_t qbytes = ((size_t)d * 4 + 15) / 16 * 16;
  int* prefix = reinterpret_cast<int*>(smem + qbytes);
  const int nseg = a.mode == 0 ? 1 : a.nprobe;
  const size_t pfbytes = ((size_t)(nseg + 1) * 4 + 15) / 16 * 16;

  for (int i = threadIdx.x; i < d; i += blockDim.x) qs[i] = a.queries[(size_t)qi * d + i];
  long long total;
  const long long* myprobes = a.mode == 1 ? a.probes + (size_t)qi * a.nprobe : nullptr;
  if (a.mode == 0) {
    total = a.n;
  } else {
    if (threadIdx.x < 32) {  // warp-chunked exclusive scan of the probed list lengths
      int carry = 0;
      for (int base = 0; base < nseg; base += 32) {
        const int p = base + threadIdx.x;
        int len = 0;
        if (p < nseg) { const long long l = myprobes[p]; len = l >= 0 ? a.list_len[l] : 0; }
        int incl = len;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, o); if ((int)threadIdx.x >= o) incl += v; }
        if (p < nseg) prefix[p] = carry + incl - len;
        carry += __shfl_sync(0xffffffffu, incl, 31);
      }
      if (threadIdx.x == 0) prefix[nseg] = carry;
    }
    __syncthreads();
    total = prefix[nseg];
  }
  sink.init(smem + qbytes + pfbytes);  // contains a barrier (also publishes qs)

  const long long r0 = total * split / a.nsplit, r1 = total * (split + 1) / a.nsplit;
  const int quad = threadIdx.x >> 2, t = threadIdx.x & 3;
  const bool vec = (d & 3) == 0;

  auto map_row = [&](long long i) -> long long {
    if (a.mode == 0) return i;
    int lo = 0, hi = nseg - 1;  // last p with prefix[p] <= i
    while (lo < hi) {
      int mid = (lo + hi + 1) >> 1;
      if (prefix[mid] <= i) lo = mid; else hi = mid - 1;
    }
    return a.list_off[myprobes[lo]] + (i - prefix[lo]);
  };

  if (r1 > r0) {
    const long long safe_row = map_row(r0);
    for (long long base = r0; base < r1; base += SCAN_QUADS) {
      sink.step(SCAN_QUADS);
      const long long i = base + quad;
      bool valid = i < r1;
      long long row = valid ? map_row(i) : safe_row;
      long long id = -1;
      if (valid) {
        id = a.ids[row];
        valid = id >= 0 && filter_pass(a.filt, id);
      }
      if (__ballot_sync(0xffffffffu, valid) == 0u) continue;  // warp-uniform skip
      if (!valid) row = safe_row;
      const float v = Dist::eval(a.vecs, row, qs, d, t, vec);
      if (valid && t == 0) sink.take(f2ord(Dist::kL2 ? v : -v), id, i);
    }
  }
  sink.finish();
}

template <class Dist>
static __device__ __forceinline__ void scan_select_body(const ScanArgs& a, unsigned char* smem, const int slot, const int split, const int qi) {
  const size_t off = ((size_t)slot * a.nsplit + split) * a.k;
  SelectSink sink(a.pool_cap, a.k, a.has_thr, a.thr_key, a.ws_kd + off, a.ws_kid + off);
  scan_rows<Dist>(a, smem, split, qi, sink);
}

// Plain launch: grid (nsplit, nq).  Mapped launch (a.qcount != NULL, the re-run of uncertified queries): a small grid in y
// strides over the *a.qcount live slots, so the usual "nothing to redo" case costs a handful of empty CTAs.
template <class Dist>
static __global__ void __launch_bounds__(SCAN_THREADS) scan_select_kernel(const ScanArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  if (!a.qcount) { scan_select_body<Dist>(a, smem, blockIdx.y, blockIdx.x, blockIdx.y); return; }
  const int n = *a.qcount;
  for (int slot = blockIdx.y; slot < n; slot += gridDim.y) {
    scan_select_body<Dist>(a, smem, slot, blockIdx.x, a.qmap[slot]);
    __syncthreads();
  }
}

// Deep top-k key pass: grid (nsplit, nqc), the keys of query blockIdx.y's candidates [r0, r1) of split blockIdx.x.
// Dynamic shared memory: scan_key_smem_bytes.
inline size_t scan_key_smem_bytes(int d, int nprobe) {
  return ((size_t)d * 4 + 15) / 16 * 16 + ((size_t)(nprobe + 1) * 4 + 15) / 16 * 16;
}
template <class Dist>
static __global__ void __launch_bounds__(SCAN_THREADS) scan_key_kernel(const ScanArgs a, const DeepKeys o) {
  extern __shared__ __align__(16) unsigned char smem[];
  DeepKeySink sink(o, blockIdx.y);
  scan_rows<Dist>(a, smem, blockIdx.x, blockIdx.y, sink);
}

// Ordered range append (b200vs_scan_range_push, VectorReader::BruteForceRangeSearch): the hits of one tile are appended
// to each query's running list in row order, until the list holds max_results.  The walk's i-th row is vecs row src(i) with
// id ids[i]: the tile's own rows (IdentityRows), or a gathered list of an index's rows (ListRows, b200vs_brute_force_range_search).  One CTA per query (blockIdx.x, so more
// than 65535 queries fit); the CTA walks the rows SCAN_QUADS at a time, one quad per row, and compacts the step's hits
// with warp ballots and a prefix over the warps.  No atomics: the result does not depend on scheduling.
struct RangeAppendArgs {
  const float* vecs;      // the rows (normalised for cosine): the [n, d] tile, or the row store a ListRows walk indexes
  const long long* ids;   // [n] the id of each row of the walk, < 0 = never a hit
  long long n;
  int d;
  const float* queries;   // [nq, d] (normalised for cosine)
  FilterDev filt;
  uint32_t thr_key;       // hit: f2ord(L2 ? dist : -ip) < thr_key (L2: dist < radius; IP: ip > 1 - radius)
  int max_results;
  float* out_dist;        // [nq, max_results] API distances
  long long* out_ids;     // [nq, max_results]
  int* counts;            // [nq] hits kept so far; read and written back by every launch
};

constexpr int RANGE_WARPS = SCAN_THREADS / 32;
// dynamic shared memory: the query (16-byte padded), then the per-warp hit counts of two steps
inline size_t range_append_smem_bytes(int d) { return ((size_t)d * 4 + 15) / 16 * 16 + 2 * RANGE_WARPS * sizeof(int); }

struct IdentityRows {
  __device__ __forceinline__ long long operator()(long long i) const { return i; }
};
struct ListRows {
  const long long* rows;
  __device__ __forceinline__ long long operator()(long long i) const { return rows[i]; }
};

template <class Dist, class Rows>
static __global__ void __launch_bounds__(SCAN_THREADS) range_append_kernel(const RangeAppendArgs a, const Rows src) {
  extern __shared__ __align__(16) unsigned char smem[];
  constexpr int kWarps = RANGE_WARPS;
  const long long qi = blockIdx.x;
  int count = a.counts[qi];
  if (count >= a.max_results) return;
  const int d = a.d;
  float* qs = reinterpret_cast<float*>(smem);
  // per-step hit count of each warp, double-buffered: one barrier per step
  int (*warp_hits)[kWarps] = reinterpret_cast<int (*)[kWarps]>(smem + ((size_t)d * 4 + 15) / 16 * 16);
  for (int i = threadIdx.x; i < d; i += blockDim.x) qs[i] = a.queries[(size_t)qi * d + i];
  __syncthreads();
  const int quad = threadIdx.x >> 2, t = threadIdx.x & 3, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool vec = (d & 3) == 0;
  float* od = a.out_dist + (size_t)qi * a.max_results;
  long long* oi = a.out_ids + (size_t)qi * a.max_results;
  int buf = 0;
  for (long long base = 0; base < a.n; base += SCAN_QUADS) {
    const long long row = base + quad;
    bool valid = row < a.n;
    long long id = -1;
    if (valid) {
      id = a.ids[row];
      valid = id >= 0 && filter_pass(a.filt, id);
    }
    bool hit = false;
    float v = 0.f;
    if (__ballot_sync(0xffffffffu, valid) != 0u) {  // warp-uniform skip
      v = Dist::eval(a.vecs, src(row < a.n ? row : base), qs, d, t, vec);
      hit = valid && f2ord(Dist::kL2 ? v : -v) < a.thr_key;
    }
    const unsigned m = __ballot_sync(0xffffffffu, hit && t == 0);  // bit 4j = row base + 8 warp + j
    if (lane == 0) warp_hits[buf][warp] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      const int c = warp_hits[buf][w];
      before += w < warp ? c : 0;
      total += c;
    }
    if (hit && t == 0) {
      const int pos = count + before + __popc(m & ((1u << lane) - 1u));
      if (pos < a.max_results) {
        od[pos] = Dist::kL2 ? v : __fsub_rn(1.0f, v);  // FillRangeSearchResult: squared L2, or 1 - ip
        oi[pos] = id;
      }
    }
    count += total;
    buf ^= 1;
    if (count >= a.max_results) break;  // block-uniform: every thread summed the same counts
  }
  if (threadIdx.x == 0) a.counts[qi] = min(count, a.max_results);
}

// Merge the per-split partial lists of each query and emit results.
//   out_dist: API semantics (L2: squared distance; IP: 1 - ip)        [nq, k] or NULL
//   out_raw : raw metric value (L2 distance or ip)                     [nq, k] or NULL
//   out_ids : ids, -1 padded                                           [nq, k]
//   out_counts: valid entries per query                                [nq] or NULL
template <bool L2>
static __global__ void __launch_bounds__(SCAN_THREADS) merge_select_kernel(const uint32_t* __restrict__ ws_kd,
                                                                    const long long* __restrict__ ws_kid, int nparts,
                                                                    int k, int pool_cap, float* out_dist, float* out_raw,
                                                                    long long* out_ids, int* out_counts,
                                                                    const int* qmap, const int* qcount) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int nslots = qcount ? *qcount : (int)gridDim.x;
  for (int slot = blockIdx.x; slot < nslots; slot += gridDim.x) {
  const int qi = qmap ? qmap[slot] : slot;
  BlockSelect sel;
  sel.init(smem, pool_cap, k);
  const long long tot = (long long)nparts * k;
  const uint32_t* kd = ws_kd + (size_t)slot * tot;
  const long long* kid = ws_kid + (size_t)slot * tot;
  if (nparts == 1) {  // already sorted: copy through
    for (int i = threadIdx.x; i < k; i += blockDim.x) { sel.kd[i] = kd[i]; sel.kid[i] = kid[i]; }
    __syncthreads();
    if (threadIdx.x == 0) {
      int c = 0;
      while (c < k && !(sel.kd[c] == KEY_SENTINEL_D && sel.kid[c] == KEY_SENTINEL_ID)) ++c;
      *sel.count = c;
    }
    __syncthreads();
  } else {
    for (long long base = 0; base < tot; base += blockDim.x) {
      sel.maybe_prune(blockDim.x);
      const long long i = base + threadIdx.x;
      if (i < tot) {
        const uint32_t dk = kd[i];
        const long long id = kid[i];
        if (!(dk == KEY_SENTINEL_D && id == KEY_SENTINEL_ID) && sel.passes(dk, id)) sel.push(dk, id);
      }
    }
    sel.prune();
  }
  const int have = *sel.count;
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    float raw = 0.f, api = 0.f;
    long long id = -1;
    if (i < have) {
      const float v = ord2f(sel.kd[i]);
      raw = L2 ? v : -v;
      api = L2 ? raw : __fsub_rn(1.0f, raw);  // FillSearchResult, vector_index_utils.cc:632-634
      id = sel.kid[i];
    }
    if (out_dist) out_dist[(size_t)qi * k + i] = api;
    if (out_raw) out_raw[(size_t)qi * k + i] = raw;
    out_ids[(size_t)qi * k + i] = id;
  }
  if (out_counts && threadIdx.x == 0) out_counts[qi] = have;
  __syncthreads();
  }
}

// k-way merge of API-semantics parts [nparts, nq, k] (multi-GPU / sibling-index merge,
// src/vector/vector_index.cc:1056-1108): ascending distance, ties -> smaller id.
static __global__ void __launch_bounds__(SCAN_THREADS) merge_api_kernel(const float* __restrict__ pd,
                                                                 const long long* __restrict__ pi, int nparts,
                                                                 long long nq, int k, int pool_cap, float* out_dist,
                                                                 long long* out_ids) {
  extern __shared__ __align__(16) unsigned char smem[];
  const long long qi = blockIdx.x;
  BlockSelect sel;
  sel.init(smem, pool_cap, k);
  const long long tot = (long long)nparts * k;
  for (long long base = 0; base < tot; base += blockDim.x) {
    sel.maybe_prune(blockDim.x);
    const long long i = base + threadIdx.x;
    if (i < tot) {
      const long long part = i / k, j = i % k;
      const size_t off = ((size_t)part * nq + qi) * k + j;
      const long long id = pi[off];
      if (id >= 0) {
        const uint32_t dk = f2ord(pd[off]);
        if (sel.passes(dk, id)) sel.push(dk, id);
      }
    }
  }
  sel.prune();
  const int have = *sel.count;
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    out_dist[(size_t)qi * k + i] = i < have ? ord2f(sel.kd[i]) : 0.f;
    out_ids[(size_t)qi * k + i] = i < have ? sel.kid[i] : -1;
  }
}

// NormalizeVectorForFaiss (src/vector/vector_index_utils.cc:480-491): n2 = <x,x> (hooked order, the engine's
// documented choice for the un-vendored faiss::fvec_norm_L2sqr); if n2 > 0 and |1-n2| > 1e-5: x /= sqrt(n2).
static __global__ void normalize_faiss_kernel(float* x, long long n, int d) {
  const long long quad = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
  const int t = threadIdx.x & 3;
  const bool valid = quad < n;
  float* row = x + (size_t)(valid ? quad : 0) * d;
  const float n2 = quad_distance<false>(row, row, d, t, (d & 3) == 0);
  if (!valid) return;
  const float kAcc = 0.00001;
  if (n2 > 0 && fabsf(__fsub_rn(1.0f, n2)) > kAcc) {
    const float nn = __fsqrt_rn(n2);
    for (int i = t; i < d; i += 4) row[i] = __fdiv_rn(row[i], nn);
  }
}

// NormalizeVectorForHnsw (src/vector/vector_index_utils.cc:493-500): sequential scalar sum.
static __global__ void normalize_hnsw_kernel(const float* x, float* out, long long n, int d) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const float* row = x + (size_t)r * d;
  float norm = 0.0f;
  for (int i = 0; i < d; ++i) norm = __fadd_rn(norm, __fmul_rn(row[i], row[i]));
  norm = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(norm), 1e-30f));
  float* o = out + (size_t)r * d;
  for (int i = 0; i < d; ++i) o[i] = __fmul_rn(row[i], norm);
}

// Append rows into arena slots: vecs[slot[i]] = src[i], ids[slot[i]] = src_ids[i], norms[slot[i]] = <x,x>.
static __global__ void scatter_rows_kernel(const float* __restrict__ src, const long long* __restrict__ src_ids,
                                    const long long* __restrict__ slots, long long n, int d, float* vecs,
                                    long long* ids, float* norms, float* row_norms) {
  const long long quad = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
  const int t = threadIdx.x & 3;
  const bool valid = quad < n;
  const float* row = src + (size_t)(valid ? quad : 0) * d;
  const float n2 = quad_distance<false>(row, row, d, t, (d & 3) == 0);
  if (!valid) return;
  const long long s = slots[quad];
  float* dst = vecs + (size_t)s * d;
  for (int i = t; i < d; i += 4) dst[i] = row[i];
  if (t == 0) { ids[s] = src_ids[quad]; if (norms) norms[s] = n2; if (row_norms) row_norms[quad] = n2; }
}

// Relocate rows (list growth / compaction): dst[dst_rows[i]] = src[src_rows[i]] for vectors, ids, norms.
static __global__ void move_rows_kernel(const float* __restrict__ svecs, const long long* __restrict__ sids,
                                 const float* __restrict__ snorms, const long long* __restrict__ src_rows,
                                 const long long* __restrict__ dst_rows, long long n, int d, float* dvecs,
                                 long long* dids, float* dnorms) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const long long sr = src_rows[w], dr = dst_rows[w];
  const float* src = svecs + (size_t)sr * d;
  float* dst = dvecs + (size_t)dr * d;
  for (int i = lane; i < d; i += 32) dst[i] = src[i];
  if (lane == 0) { dids[dr] = sids[sr]; if (dnorms) dnorms[dr] = snorms[sr]; }
}

static __global__ void set_ids_kernel(long long* ids, const long long* slots, long long n, long long value) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ids[slots[i]] = value;
}

static __global__ void iota_kernel(long long* p, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = i;
}

}  // namespace b200vs
