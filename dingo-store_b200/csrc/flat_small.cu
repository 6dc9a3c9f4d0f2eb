// flat_small.cu — exact Flat search for tiny batches (nq < 16; the reference's own execution shape is ONE query per task,
// src/vector/vector_index.cc:54 + :244-271, and BASELINE config 1 is quoted at batch 1).
//
// The general exact path (scan_select_kernel + merge_select_kernel) spends two launches and a block-wide pool select on
// what is, for one query over 100 K x 128 floats, a 51 MB stream (15 us at an H100's 3.35 TB/s).  Here ONE launch covers it:
//   * grid = (row slices, queries): ~2 CTAs per SM, each CTA streams its slice of the database once (quads of 4 threads per
//     row, 128-bit loads, the reference's AVX-512 summation order -> bit-identical distances), stores its (key, id) pairs in
//     shared memory, and one warp selects the slice's top-k with a warp-level radix select + rank sort (no block-wide sort);
//   * the CTA that finishes last (atomic ticket) merges the per-slice top-k lists of its query the same way and writes the
//     API-semantics result: the cross-CTA top-k needs no second launch.
// Ties: (distance, id) order like every other path, mass duplicates included (fs_topk_warp).
//
// Replaces faiss exhaustive_{L2sqr,inner_product}_seq + HeapBlockResultHandler behind VectorIndexFlat::Search
// (src/vector/vector_index_flat.cc:249-252) for nq < 16.
#include <atomic>
#include <cstdio>
#include <cstdlib>

#include "flat_small.cuh"
#include "scan_kernels.cuh"
#include "warp_select.cuh"

namespace b200vs {

constexpr int FS_THREADS = 512;
constexpr int FS_PAIRS = 3072;  // (key, id) pairs a CTA holds in shared memory: its slice's rows, later the per-slice lists it merges
constexpr int FS_CT = 128;      // entries the rank sort holds (k <= FS_CT / 2)

struct FsArgs {
  const float* vecs;
  const long long* ids;
  const float* queries;  // [nq, d]
  int d;
  long long n;
  int rows_per_cta;
  int k;
  FilterDev filt;
  uint32_t* part_kd;     // [nq, nslices, k]
  long long* part_id;    // [nq, nslices, k]
  int* tickets;          // [nq] zeroed before the launch
  uint32_t* gthr_inv;    // [nq] zeroed: ~(smallest k-th key any slice has published) — an upper bound of the global k-th key
  float* out_dist;       // [nq, k] API semantics, or the raw metric value (L2 distance | ip) when raw_out
  long long* out_ids;    // [nq, k]
  long long* dbg;        // optional [8] clock64 stamps of slice 0 and of the merging CTA (B200VS_FS_DEBUG)
  int raw_out;
};

__device__ __forceinline__ long long warp_min_ll(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const long long w = __shfl_xor_sync(0xffffffffu, v, o); v = w < v ? w : v; }
  return v;
}

// top-k (ascending (key, id)) of n (key, id) pairs in shared memory, by ALL threads of the CTA; emit(rank, kd, id) receives
// the result; returns how many live pairs were emitted.  Usual case: the k-th key kth comes from a block-wide radix select and
// the <= FS_CT pairs with key <= kth are rank-sorted.  Mass ties (more than FS_CT pairs share the k-th key: duplicated
// vectors): the pairs strictly below kth are kept and the open slots are filled with the smallest ids among the tied pairs,
// one warp-min per slot (warp 0) — same (key, id) order, no limit on the number of duplicates.
struct FsShared {
  BlockSelShared sel;
  uint32_t ckd[FS_CT];
  long long cid[FS_CT];
  int m;
};
template <class Emit>
__device__ __forceinline__ int fs_topk_block(const uint32_t* kd, const long long* id, int n, int k, FsShared& F, Emit emit) {
  const int lane = threadIdx.x & 31;
  if (n <= FS_CT) {  // a handful of pairs (the pruned merge): every thread ranks its pair against all others — n^2 compares, only worth it when tiny
    if (threadIdx.x == 0) F.m = 0;
    __syncthreads();
    int live = 0;
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
      const uint32_t d0 = kd[e];
      const long long i0 = id[e];
      if (d0 == KEY_SENTINEL_D && i0 == KEY_SENTINEL_ID) continue;
      ++live;
      int rank = 0;
      for (int j = 0; j < n; ++j) {
        const uint32_t dj = kd[j];
        const long long ij = id[j];
        rank += (key_less(dj, ij, d0, i0) || (dj == d0 && ij == i0 && j < e)) ? 1 : 0;  // (sentinel pairs rank last)
      }
      if (rank < k) emit(rank, d0, i0);
    }
    live = __reduce_add_sync(0xffffffffu, live);
    if (lane == 0 && live) atomicAdd(&F.m, live);
    __syncthreads();
    return min(F.m, k);
  }
  uint32_t kth = 0xFFFFFFFFu;
  if (n > k) kth = block_kth_key_any(k, F.sel, [&](auto f) { for (int i = threadIdx.x; i < n; i += blockDim.x) f(kd[i]); });
  if (threadIdx.x == 0) F.m = 0;
  __syncthreads();
  for (int base = 0; base < n; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const bool in = i < n && kd[i] <= kth && !(kd[i] == KEY_SENTINEL_D && id[i] == KEY_SENTINEL_ID);  // empty slots never surface
    const unsigned msk = __ballot_sync(0xffffffffu, in);
    int wbase = 0;
    if (lane == 0 && msk) wbase = atomicAdd(&F.m, __popc(msk));
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    const int p = wbase + __popc(msk & ((1u << lane) - 1u));
    if (in && p < FS_CT) { F.ckd[p] = kd[i]; F.cid[p] = id[i]; }
  }
  __syncthreads();
  int m = F.m;
  if (m > FS_CT) {  // mass ties at the k-th key: warp 0 resolves them
    __syncthreads();
    if (threadIdx.x < 32) {
      m = 0;
      for (int base = 0; base < n; base += 32) {
        const int i = base + lane;
        const bool in = i < n && kd[i] < kth;
        const unsigned msk = __ballot_sync(0xffffffffu, in);
        if (in) { const int p = m + __popc(msk & ((1u << lane) - 1u)); F.ckd[p] = kd[i]; F.cid[p] = id[i]; }  // fewer than k such pairs
        m += __popc(msk);
      }
      long long last = (long long)0x8000000000000000LL;
      for (; m < k; ++m) {
        long long best = KEY_SENTINEL_ID;
        for (int i = lane; i < n; i += 32) if (kd[i] == kth && id[i] > last && id[i] < best) best = id[i];
        best = warp_min_ll(best);
        if (best == KEY_SENTINEL_ID) break;
        if (lane == 0) { F.ckd[m] = kth; F.cid[m] = best; }
        last = best;
      }
      if (lane == 0) F.m = m;
    }
    __syncthreads();
    m = F.m;
  }
  block_rank_sort(F.ckd, F.cid, m, [&](int rank, int e) { if (rank < k) emit(rank, F.ckd[e], F.cid[e]); });
  return min(m, k);
}

template <bool L2>
static __global__ void __launch_bounds__(FS_THREADS) flat_small_kernel(const FsArgs a) {
  extern __shared__ __align__(16) unsigned char fs_smem[];  // [FS_PAIRS] ids, [FS_PAIRS] keys, then the query row
  __shared__ FsShared F;
  __shared__ int s_n, s_last;
  long long* s_id = reinterpret_cast<long long*>(fs_smem);
  uint32_t* s_kd = reinterpret_cast<uint32_t*>(fs_smem + (size_t)FS_PAIRS * 8);
  float* qs = reinterpret_cast<float*>(fs_smem + (size_t)FS_PAIRS * 12);
  const int qi = blockIdx.y, slice = blockIdx.x, nslices = gridDim.x;
  const int d = a.d, k = a.k;
  const long long t_start = clock64();
  for (int i = threadIdx.x; i < d; i += FS_THREADS) qs[i] = a.queries[(size_t)qi * d + i];
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  const long long r0 = (long long)slice * a.rows_per_cta, r1 = min(a.n, r0 + a.rows_per_cta);
  const int quad = threadIdx.x >> 2, t = threadIdx.x & 3;
  const bool vec = (d & 3) == 0;
  for (long long base = r0; base < r1; base += FS_THREADS / 4) {
    const long long row = base + quad;
    bool valid = row < r1;
    long long id = -1;
    if (valid) { id = a.ids[row]; valid = id >= 0 && filter_pass(a.filt, id); }
    if (__ballot_sync(0xffffffffu, valid) == 0u) continue;
    const float v = quad_distance<L2>(a.vecs + (size_t)(valid ? row : r0) * d, qs, d, t, vec);
    const unsigned wm = __ballot_sync(0xffffffffu, valid && t == 0);  // one shared-memory atomic per warp
    int wbase = 0;
    if ((threadIdx.x & 31) == 0) wbase = atomicAdd(&s_n, __popc(wm));
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    if (valid && t == 0) { const int p = wbase + __popc(wm & ((1u << (threadIdx.x & 31)) - 1u)); s_kd[p] = f2ord(L2 ? v : -v); s_id[p] = id; }
  }
  __syncthreads();
  const long long t_scan = clock64();
  uint32_t* pk = a.part_kd + ((size_t)qi * nslices + slice) * k;
  long long* pi = a.part_id + ((size_t)qi * nslices + slice) * k;
  {
    const int n = s_n;
    const int have = fs_topk_block(s_kd, s_id, n, k, F, [&](int rank, uint32_t kd, long long id) {
      pk[rank] = kd; pi[rank] = id;
      if (rank == k - 1) atomicMax(a.gthr_inv + qi, ~kd);  // this slice alone holds k rows at or below kd: the global k-th key is <= kd
    });
    for (int i = have + (int)threadIdx.x; i < k; i += FS_THREADS) { pk[i] = KEY_SENTINEL_D; pi[i] = KEY_SENTINEL_ID; }
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      s_last = atomicAdd(a.tickets + qi, 1) == nslices - 1 ? 1 : 0;
    }
  }
  __syncthreads();
  if (a.dbg && slice == 0 && threadIdx.x == 0) { a.dbg[0] = t_scan - t_start; a.dbg[1] = clock64() - t_scan; }
  if (!s_last) return;
  const long long t_merge0 = clock64();
  // ---- the CTA that finished last merges the per-slice lists of this query: no second launch ----
  __threadfence();
  const int tot = nslices * k;  // <= FS_PAIRS (launcher)
  const uint32_t* allk = a.part_kd + (size_t)qi * nslices * k;
  const long long* alli = a.part_id + (size_t)qi * nslices * k;
  // only pairs at or below the tightest published k-th key can be among the global top-k: a few dozen of the nslices * k
  const uint32_t thr = ~__ldcg(a.gthr_inv + qi);
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  for (int base = 0; base < tot; base += FS_THREADS) {
    const int j = base + threadIdx.x;
    uint32_t kd = KEY_SENTINEL_D;
    long long id = KEY_SENTINEL_ID;
    if (j < tot) { kd = __ldcg(allk + j); id = __ldcg(alli + j); }
    const bool in = kd <= thr && !(kd == KEY_SENTINEL_D && id == KEY_SENTINEL_ID);
    const unsigned msk = __ballot_sync(0xffffffffu, in);
    int wbase = 0;
    if ((threadIdx.x & 31) == 0 && msk) wbase = atomicAdd(&s_n, __popc(msk));
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    if (in) { const int p = wbase + __popc(msk & ((1u << (threadIdx.x & 31)) - 1u)); s_kd[p] = kd; s_id[p] = id; }
  }
  __syncthreads();
  {
    const int n = s_n;
    const int have = fs_topk_block(s_kd, s_id, n, k, F, [&](int rank, uint32_t kd, long long id) {
      const float v = ord2f(kd);
      const float raw = L2 ? v : -v;
      a.out_dist[(size_t)qi * k + rank] = (L2 || a.raw_out) ? raw : __fsub_rn(1.0f, raw);
      a.out_ids[(size_t)qi * k + rank] = id;
    });
    for (int i = have + (int)threadIdx.x; i < k; i += FS_THREADS) { a.out_dist[(size_t)qi * k + i] = 0.f; a.out_ids[(size_t)qi * k + i] = -1; }
    if (a.dbg && threadIdx.x == 0) { a.dbg[2] = clock64() - t_merge0; a.dbg[3] = t_merge0 - t_start; a.dbg[4] = slice; }
  }
}

constexpr int FS_MAX_D = 2048;
constexpr size_t FS_MAX_SMEM = (size_t)FS_PAIRS * 12 + (size_t)FS_MAX_D * 4;  // pair buffer + query row: 44 KB at d = 2048

// The pair buffer (36 KB) plus a query row of up to 8 KB is requested as dynamic shared memory; with the kernel's ~6 KB of
// static shared memory that passes the 48 KB a launch gets without opting in once d > 1592.  Both instantiations are opted
// in to the largest request once per device.
static void fs_opt_in(int device) {
  static std::atomic<bool> done[64];
  const bool cached = device >= 0 && device < 64;
  if (cached && done[device].load(std::memory_order_acquire)) return;
  B200VS_CUDA(cudaFuncSetAttribute(flat_small_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FS_MAX_SMEM));
  B200VS_CUDA(cudaFuncSetAttribute(flat_small_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FS_MAX_SMEM));
  if (cached) done[device].store(true, std::memory_order_release);
}

bool flat_small_eligible(int device, int64_t nq, int64_t n, int d, int k, const SearchCtx& sc) {
  if (sc.exact_only) return false;              // "exact_only" callers ask for the general path explicitly (tests compare the two)
  if (nq < 1 || nq >= 16 || n < 4096) return false;
  if (2 * k > FS_CT || d > FS_MAX_D) return false;  // rank-sort buffer; pair buffer + query row = FS_MAX_SMEM (launcher opts in past 48 KB)
  if (nq > 4 && (double)n * d * 4 > 40e6) return false;  // more than a few queries re-stream the table: only while it stays in L2 (50 MB on an H100)
  const int nslices = std::min(2 * device_sm_count(device), FS_PAIRS / std::max(1, k));
  return cdiv(n, nslices) <= FS_PAIRS;          // a slice's rows must fit the pair buffer (tables beyond ~900 K rows: general path)
}

void flat_small_search(IndexBase* ix, bool l2, const float* vecs, const long long* ids, int64_t n, int64_t nq, const float* q, int k,
                       const SearchCtx& sc, float* out_dist, long long* out_ids, bool raw_out, cudaStream_t s) {
  const int d = ix->dim;
  // ~2 CTAs per SM per query, bounded so that the final merge (nslices * k pairs) fits the pair buffer
  int nslices = (int)std::min<int64_t>(std::min(2 * device_sm_count(ix->device), FS_PAIRS / std::max(1, k)), std::max<int64_t>(1, n / 64));
  const int rows = (int)cdiv(n, nslices);
  if (rows > FS_PAIRS) fail(B200VS_EINTERNAL, "flat_small_search called on an ineligible shape");
  nslices = (int)cdiv(n, rows);
  auto& S = ix->scratch;
  FsArgs a;
  a.vecs = vecs; a.ids = ids; a.queries = q; a.d = d; a.n = n; a.rows_per_cta = rows; a.k = k;
  a.filt.has_range = sc.has_range; a.filt.negate = sc.negate; a.filt.rmin = sc.rmin; a.filt.rmax = sc.rmax;
  a.filt.sorted_ids = sc.sorted_ids_dev; a.filt.n_ids = sc.n_ids;
  a.part_kd = S.alloc<uint32_t>((size_t)nq * nslices * k);
  a.part_id = S.alloc<long long>((size_t)nq * nslices * k);
  a.tickets = S.alloc<int>(2 * nq);
  a.gthr_inv = reinterpret_cast<uint32_t*>(a.tickets + nq);
  a.out_dist = out_dist; a.out_ids = out_ids; a.raw_out = raw_out ? 1 : 0;
  static const bool debug = getenv("B200VS_FS_DEBUG") != nullptr;
  a.dbg = debug ? S.alloc<long long>(8) : nullptr;
  B200VS_CUDA(cudaMemsetAsync(a.tickets, 0, (size_t)nq * 8, s));
  const size_t smem = (size_t)FS_PAIRS * 12 + ((size_t)d * 4 + 15) / 16 * 16;
  if (smem > FS_MAX_SMEM) fail(B200VS_EINTERNAL, "flat_small_search called on an ineligible dimension");
  fs_opt_in(ix->device);
  dim3 grid(nslices, (unsigned)nq);
  if (l2) flat_small_kernel<true><<<grid, FS_THREADS, smem, s>>>(a);
  else flat_small_kernel<false><<<grid, FS_THREADS, smem, s>>>(a);
  B200VS_CUDA(cudaGetLastError());
  ix->launch_count(1);
  if (debug) {
    long long h[8] = {0};
    B200VS_CUDA(cudaMemcpyAsync(h, a.dbg, 40, cudaMemcpyDeviceToHost, s));
    B200VS_CUDA(cudaStreamSynchronize(s));
    fprintf(stderr, "[b200vs] flat_small: slice0 scan %lld clk, select+ticket %lld clk; merging CTA (slice %lld): started merge at +%lld clk, merge %lld clk; grid %d x %d, %d rows/CTA\n",
            h[0], h[1], h[4], h[3], h[2], nslices, (int)nq, rows);
  }
}

}  // namespace b200vs
