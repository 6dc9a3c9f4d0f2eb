// brute_force.cu — b200vs_brute_force_search / b200vs_brute_force_range_search: VectorReader::BruteForceSearch and
// BruteForceRangeSearch (src/vector/vector_reader.cc:1873-2202) answered from an index's own device rows instead of a
// RocksDB scan whose rows are pushed through b200vs_scan_* / b200vs_scan_range_*, with the results those scans give for the
// index's live rows fed in ascending id order.
#include <thrust/iterator/counting_iterator.h>

#include <cub/cub.cuh>

#include "filter.cuh"
#include "index.h"
#include "ivf_common.h"
#include "tc_scan.cuh"

namespace b200vs {

namespace {

// one CTA per list: the ids of its rows [off, off + len); every other row of the arena was set to -1 before
__global__ void list_ids_kernel(const long long* __restrict__ ids, const long long* __restrict__ off, const int* __restrict__ len,
                                long long* __restrict__ out) {
  const long long o = off[blockIdx.x];
  const int n = len[blockIdx.x];
  for (int i = threadIdx.x; i < n; i += blockDim.x) out[o + i] = ids[o + i];
}

__global__ void node_ids_kernel(const long long* __restrict__ labels, const unsigned char* __restrict__ deleted, long long n,
                                long long* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = deleted[i] ? -1 : labels[i];
}

// a row the range search walks: a live id that passes the filters
struct LiveRow {
  const long long* ids;
  FilterDev f;
  __device__ __forceinline__ bool operator()(long long r) const {
    const long long id = ids[r];
    return id >= 0 && filter_pass(f, id);
  }
};

__global__ void gather_ids_kernel(const long long* __restrict__ ids, const long long* __restrict__ rows, long long n,
                                  long long* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = ids[rows[i]];
}

}  // namespace

void launch_list_ids(const long long* ids, const long long* off, const int* len, int nlist, int64_t rows, long long* out,
                     cudaStream_t s) {
  B200VS_CUDA(cudaMemsetAsync(out, 0xFF, (size_t)rows * 8, s));
  list_ids_kernel<<<(unsigned)nlist, 256, 0, s>>>(ids, off, len, out);
  B200VS_CUDA(cudaGetLastError());
}

void launch_node_ids(const long long* labels, const unsigned char* deleted, int64_t n, long long* out, cudaStream_t s) {
  node_ids_kernel<<<(unsigned)cdiv(n, 256), 256, 0, s>>>(labels, deleted, n, out);
  B200VS_CUDA(cudaGetLastError());
}

// Top-k is order-free: one search of the Flat view of every row slot.  b200vs_scan_push merges each tile's results into the
// running top-k by (API distance, id), so for IP / cosine, where 1 - ip can round two raw values to one distance, the
// results are ordered by that merge's rule once more; for L2 the search's own order is that order.
// Range keeps the first max_results hits in ascending id order: one compaction of the live rows that pass the filters
// into (row) in storage order, one stable sort of (id, row) by id (rows sharing an id, which an IVF index may hold, stay in
// storage order), then range_append_kernel walks the rows through that list.
void brute_force(IndexBase* ix, const SearchReq& r, cudaStream_t s) {
  TcView v;
  if (!ix->brute_force_rows(v, !r.range && r.nq >= 16, s)) { fill_empty(r, s); return; }
  auto& S = ix->scratch;
  if (!r.range) {
    if (ix->metric == B200VS_L2) { flat_view_search(ix, v, r, s); return; }
    SearchReq t = r;
    t.od = S.alloc<float>((size_t)r.nq * r.k);
    t.oi = S.alloc<long long>((size_t)r.nq * r.k);
    flat_view_search(ix, v, t, s);
    if (r.deep) run_deep_merge_api(ix, r.nq, r.k, r.k, t.od, t.oi, r.od, r.oi, s);
    else launch_merge_api(1, r.nq, r.k, t.od, t.oi, r.od, r.oi, s);
    ix->launch_count(1);
    return;
  }
  const int64_t n = v.arena_rows;
  if (n >= (1LL << 31)) fail(B200VS_EILLEGAL_PARAMETERS, "brute-force range search holds at most 2^31 - 1 row slots");
  const SearchCtx& sc = *r.sc;
  const float* q = ix->queries(r, s);
  B200VS_CUDA(cudaMemsetAsync(r.od, 0, (size_t)r.nq * r.k * 4, s));
  B200VS_CUDA(cudaMemsetAsync(r.oi, 0xFF, (size_t)r.nq * r.k * 8, s));  // id -1 = empty slot
  B200VS_CUDA(cudaMemsetAsync(r.oc, 0, (size_t)r.nq * 4, s));
  LiveRow live{v.ids, FilterDev{}};
  live.f.has_range = sc.has_range; live.f.negate = sc.negate; live.f.rmin = sc.rmin; live.f.rmax = sc.rmax;
  live.f.sorted_ids = sc.sorted_ids_dev; live.f.n_ids = sc.n_ids;
  long long* rows = S.alloc<long long>(n);
  int* d_m = S.alloc<int>(1);
  const thrust::counting_iterator<long long> all(0);
  size_t tmp_bytes = 0;
  B200VS_CUDA(cub::DeviceSelect::If(nullptr, tmp_bytes, all, rows, d_m, (int)n, live, s));
  B200VS_CUDA(cub::DeviceSelect::If(S.alloc<unsigned char>(std::max<size_t>(tmp_bytes, 1)), tmp_bytes, all, rows, d_m, (int)n, live, s));
  int m = 0;
  B200VS_CUDA(cudaMemcpyAsync(&m, d_m, 4, cudaMemcpyDeviceToHost, s));
  B200VS_CUDA(cudaStreamSynchronize(s));
  ix->launch_count(1);
  if (m == 0) return;
  long long* keys = S.alloc<long long>(m);
  long long* ids = S.alloc<long long>(m);
  long long* order = S.alloc<long long>(m);
  gather_ids_kernel<<<(unsigned)cdiv(m, 256), 256, 0, s>>>(v.ids, rows, m, keys);
  B200VS_CUDA(cudaGetLastError());
  sort_by_id(m, keys, ids, rows, order, [&](size_t bytes) -> void* { return S.alloc<unsigned char>(std::max<size_t>(bytes, 1)); }, s);
  const float thr = ix->ip_like() ? 1.0F - r.radius : r.radius;
  launch_range_append(ix->metric == B200VS_L2, v.vecs, ids, order, m, ix->dim, r.nq, q, sc, thr, r.k, r.od, r.oi, r.oc, s);
  ix->launch_count(3);
}

}  // namespace b200vs
