// kernels.cu — launchers of the exact scan/select kernels (scan_kernels.cuh).
#include <algorithm>

#include "index.h"
#include "ivf_common.h"
#include "scan_kernels.cuh"

namespace b200vs {

static constexpr int kMaxDynSmem = 227 * 1024;

template <class K>
static void ensure_smem(K kernel, size_t bytes) {
  if (bytes > (size_t)kMaxDynSmem) fail(B200VS_EILLEGAL_PARAMETERS, "request needs more shared memory than one SM has (topk/nprobe/dimension too large)");
  // raise the opt-in limit once per kernel (cheap, idempotent)
  B200VS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
}

static void run_scan_impl(IndexBase* ix, const ScanJob& job, int64_t nq, const float* queries, int k, float* out_dist,
                          float* out_raw, long long* out_ids, int* out_counts, const int* qmap, const int* qcount,
                          int forced_nsplit, cudaStream_t s);

// the rows, candidate space and filters of job's scan
static ScanArgs scan_args(const ScanJob& job, const float* queries) {
  ScanArgs a{};
  a.vecs = job.vecs; a.ids = job.ids; a.queries = queries; a.d = job.d; a.mode = job.mode; a.n = job.n;
  a.probes = job.probes; a.nprobe = job.nprobe; a.list_off = job.list_off; a.list_len = job.list_len;
  a.filt.has_range = job.sc ? job.sc->has_range : 0;
  a.filt.negate = job.sc ? job.sc->negate : 0;
  a.filt.rmin = job.sc ? job.sc->rmin : 0;
  a.filt.rmax = job.sc ? job.sc->rmax : 0;
  a.filt.sorted_ids = job.sc ? job.sc->sorted_ids_dev : nullptr;
  a.filt.n_ids = job.sc ? job.sc->n_ids : 0;
  return a;
}

template <class Dist>
static void launch_scan_keys(const ScanArgs& a, dim3 grid, size_t smem, const DeepKeys& o, cudaStream_t s) {
  ensure_smem(scan_key_kernel<Dist>, smem);
  scan_key_kernel<Dist><<<grid, SCAN_THREADS, smem, s>>>(a, o);
  B200VS_CUDA(cudaGetLastError());
}

bool exact_select_fits(int d, int nseg, int k) {
  return scan_smem_bytes(d, nseg, select_pool_cap(k, SCAN_THREADS)) <= (size_t)kMaxDynSmem;
}

// Deep top-k over the exact scan: its key pass runs scan_rows with DeepKeySink, each query's candidates split over enough CTAs
// to fill the SMs (a CTA holds no select pool, so the split costs nothing but the query load)
void run_scan_deep(IndexBase* ix, const ScanJob& job, int64_t nq, const float* queries, int k, float* od, bool raw, long long* oi,
                   cudaStream_t s) {
  DeepJob dj;
  dj.l2 = job.l2; dj.mode = job.mode; dj.n = job.n; dj.ids = job.ids;
  dj.probes = job.probes; dj.nprobe = job.nprobe; dj.list_off = job.list_off; dj.list_len = job.list_len;
  const ScanArgs base = scan_args(job, queries);
  const size_t smem = scan_key_smem_bytes(job.d, job.mode == 0 ? 1 : job.nprobe);
  const int sms = device_sm_count(ix->device);
  run_deep(ix, dj, nq, k, od, raw, oi, [&](int64_t q0, int nqc, const DeepKeys& o, cudaStream_t st) {
    ScanArgs a = base;
    a.queries = queries + (size_t)q0 * job.d;
    if (job.mode == 1) a.probes = job.probes + (size_t)q0 * job.nprobe;
    a.nsplit = (int)std::max<int64_t>(1, std::min<int64_t>(cdiv(o.stride, 4096), std::max(1, sms * 8 / nqc)));
    const dim3 grid(a.nsplit, nqc);
    if (job.hamming) launch_scan_keys<HammingDist>(a, grid, smem, o, st);
    else if (job.l2) launch_scan_keys<Fp32Dist<true>>(a, grid, smem, o, st);
    else launch_scan_keys<Fp32Dist<false>>(a, grid, smem, o, st);
    ix->launch_count(1);
  }, s);
}

void run_scan(IndexBase* ix, const ScanJob& job, int64_t nq, const float* queries, int k, float* out_dist,
              float* out_raw, long long* out_ids, int* out_counts, cudaStream_t s) {
  run_scan_impl(ix, job, nq, queries, k, out_dist, out_raw, out_ids, out_counts, nullptr, nullptr, 0, s);
}

// exact re-run of the queries listed in qmap[0 .. *qcount) (device-side count; grid sized for nq_max)
void run_scan_mapped(IndexBase* ix, const ScanJob& job, int64_t nq_max, const int* qmap, const int* qcount, const float* queries,
                     int k, float* out_dist, float* out_raw, long long* out_ids, int* out_counts, cudaStream_t s) {
  // few queries are ever re-run, but each one re-streams all its candidates: split a query over enough CTAs that a single
  // flagged query of a large index (cfg5: 2.4 GB of probed rows) is not an 8-CTA, 50 ms affair
  const double cand = job.mode == 0 ? (double)job.n : job.avg_candidates;
  int nsplit = (int)std::max(8.0, std::min(128.0, cand / 512.0));
  nsplit = (int)std::max<int64_t>(8, std::min<int64_t>(nsplit, (64LL << 20) / std::max<int64_t>(1, nq_max * k)));  // partial-result workspace
  run_scan_impl(ix, job, nq_max, queries, k, out_dist, out_raw, out_ids, out_counts, qmap, qcount, nsplit, s);
}

static void run_scan_impl(IndexBase* ix, const ScanJob& job, int64_t nq, const float* queries, int k, float* out_dist,
                          float* out_raw, long long* out_ids, int* out_counts, const int* qmap, const int* qcount,
                          int forced_nsplit, cudaStream_t s) {
  if (nq <= 0 || k <= 0) return;
  if (nq > 65535) fail(B200VS_EILLEGAL_PARAMETERS, "batch too large (max 65535 queries per call)");
  // split each query's candidate range over several CTAs when the batch alone cannot fill the SMs
  const int target_blocks = device_sm_count(ix->device) * 4;
  int nsplit = (int)std::max<int64_t>(1, (target_blocks + nq - 1) / nq);
  const double cand = job.mode == 0 ? (double)job.n : job.avg_candidates;
  const int max_by_work = (int)std::max(1.0, cand / 512.0);
  nsplit = std::max(1, std::min(nsplit, std::min(max_by_work, 128)));
  if (forced_nsplit > 0) nsplit = forced_nsplit;

  const int cap = select_pool_cap(k, SCAN_THREADS);  // SCAN_THREADS >= SCAN_QUADS: one size for both kernels
  ScanArgs a = scan_args(job, queries);
  a.k = k; a.nsplit = nsplit;
  a.ws_kd = ix->scratch.alloc<uint32_t>((size_t)nq * nsplit * k);
  a.ws_kid = ix->scratch.alloc<long long>((size_t)nq * nsplit * k);
  a.has_thr = job.has_thr ? 1 : 0;
  a.thr_key = job.has_thr ? f2ord(job.l2 ? job.thr_raw : -job.thr_raw) : 0;
  a.pool_cap = cap;
  a.qmap = qmap; a.qcount = qcount;

  const size_t smem1 = scan_smem_bytes(job.d, job.mode == 0 ? 1 : job.nprobe, cap);
  const size_t smem2 = BlockSelect::smem_bytes(cap);
  // mapped launch: a fixed budget of ~4 CTAs per SM strides over the live slots (the usual "nothing to redo" launch stays cheap)
  const unsigned slots = qcount ? (unsigned)std::min<int64_t>(nq, std::max(1, 592 / nsplit)) : (unsigned)nq;
  dim3 grid(nsplit, slots);
  ScopedKernelTimer timer(ix, s, ix->profiling && job.dominant);
  if (job.hamming) {
    ensure_smem(scan_select_kernel<HammingDist>, smem1);
    scan_select_kernel<HammingDist><<<grid, SCAN_THREADS, smem1, s>>>(a);
    timer.stop();
    ensure_smem(merge_select_kernel<true>, smem2);
    merge_select_kernel<true><<<slots, SCAN_THREADS, smem2, s>>>(a.ws_kd, a.ws_kid, nsplit, k, cap, out_dist, out_raw, out_ids, out_counts, qmap, qcount);
  } else if (job.l2) {
    ensure_smem(scan_select_kernel<Fp32Dist<true>>, smem1);
    scan_select_kernel<Fp32Dist<true>><<<grid, SCAN_THREADS, smem1, s>>>(a);
    timer.stop();
    ensure_smem(merge_select_kernel<true>, smem2);
    merge_select_kernel<true><<<slots, SCAN_THREADS, smem2, s>>>(a.ws_kd, a.ws_kid, nsplit, k, cap, out_dist, out_raw, out_ids, out_counts, qmap, qcount);
  } else {
    ensure_smem(scan_select_kernel<Fp32Dist<false>>, smem1);
    scan_select_kernel<Fp32Dist<false>><<<grid, SCAN_THREADS, smem1, s>>>(a);
    timer.stop();
    ensure_smem(merge_select_kernel<false>, smem2);
    merge_select_kernel<false><<<slots, SCAN_THREADS, smem2, s>>>(a.ws_kd, a.ws_kid, nsplit, k, cap, out_dist, out_raw, out_ids, out_counts, qmap, qcount);
  }
  B200VS_CUDA(cudaGetLastError());
  ix->launch_count(2);
}

template <class Dist, class Rows>
static void launch_range_append_rows(const RangeAppendArgs& a, int64_t nq, const Rows& src, cudaStream_t s) {
  const size_t smem = range_append_smem_bytes(a.d);
  ensure_smem(range_append_kernel<Dist, Rows>, smem);
  range_append_kernel<Dist, Rows><<<(unsigned)nq, SCAN_THREADS, smem, s>>>(a, src);
}

void launch_range_append(bool l2, const float* vecs, const long long* ids, const long long* rows, int64_t n, int d, int64_t nq,
                         const float* queries, const SearchCtx& sc, float thr_raw, int max_results, float* out_dist,
                         long long* out_ids, int* counts, cudaStream_t s) {
  if (n <= 0 || nq <= 0) return;
  RangeAppendArgs a;
  a.vecs = vecs; a.ids = ids; a.n = n; a.d = d; a.queries = queries;
  a.filt.has_range = sc.has_range; a.filt.negate = sc.negate; a.filt.rmin = sc.rmin; a.filt.rmax = sc.rmax;
  a.filt.sorted_ids = sc.sorted_ids_dev; a.filt.n_ids = sc.n_ids;
  a.thr_key = f2ord(l2 ? thr_raw : -thr_raw);
  a.max_results = max_results; a.out_dist = out_dist; a.out_ids = out_ids; a.counts = counts;
  if (rows) {
    const ListRows src{rows};
    if (l2) launch_range_append_rows<Fp32Dist<true>>(a, nq, src, s);
    else launch_range_append_rows<Fp32Dist<false>>(a, nq, src, s);
  } else {
    if (l2) launch_range_append_rows<Fp32Dist<true>>(a, nq, IdentityRows{}, s);
    else launch_range_append_rows<Fp32Dist<false>>(a, nq, IdentityRows{}, s);
  }
  B200VS_CUDA(cudaGetLastError());
}

__global__ void mark_probed_kernel(const long long* probes, long long n, int* flags) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && probes[i] >= 0) flags[probes[i]] = 1;
}
__global__ void sum_probed_kernel(const int* flags, const int* list_len, int nlist, unsigned long long* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nlist && flags[i]) { atomicAdd(out, (unsigned long long)list_len[i]); atomicAdd(out + 1, 1ULL); }
}
void profile_probed(IndexBase* ix, const long long* probes, int64_t n_probes, int nlist, const int* list_len, cudaStream_t s) {
  int* flags = ix->scratch.alloc<int>(nlist);
  unsigned long long* out = ix->scratch.alloc<unsigned long long>(2);
  B200VS_CUDA(cudaMemsetAsync(flags, 0, (size_t)nlist * 4, s));
  B200VS_CUDA(cudaMemsetAsync(out, 0, 16, s));
  mark_probed_kernel<<<(unsigned)cdiv(n_probes, 256), 256, 0, s>>>(probes, n_probes, flags);
  sum_probed_kernel<<<(unsigned)cdiv(nlist, 256), 256, 0, s>>>(flags, list_len, nlist, out);
  unsigned long long h[2];
  B200VS_CUDA(cudaMemcpyAsync(h, out, 16, cudaMemcpyDeviceToHost, s));
  B200VS_CUDA(cudaStreamSynchronize(s));
  ix->stats[4] = (int64_t)h[0];
  ix->stats[5] = (int64_t)h[1];
}

void launch_normalize_faiss(float* x, int64_t n, int d, cudaStream_t s) {
  if (n <= 0) return;
  const int threads = 256;
  const int64_t blocks = cdiv(n * 4, threads);
  normalize_faiss_kernel<<<(unsigned)blocks, threads, 0, s>>>(x, n, d);
  B200VS_CUDA(cudaGetLastError());
}
void launch_normalize_hnsw(const float* x, float* out, int64_t n, int d, cudaStream_t s) {
  if (n <= 0) return;
  normalize_hnsw_kernel<<<(unsigned)cdiv(n, 128), 128, 0, s>>>(x, out, n, d);
  B200VS_CUDA(cudaGetLastError());
}
void launch_scatter_rows(const float* src, const long long* src_ids, const long long* slots, int64_t n, int d,
                         float* vecs, long long* ids, float* norms, float* row_norms, cudaStream_t s) {
  if (n <= 0) return;
  const int threads = 256;
  scatter_rows_kernel<<<(unsigned)cdiv(n * 4, threads), threads, 0, s>>>(src, src_ids, slots, n, d, vecs, ids, norms, row_norms);
  B200VS_CUDA(cudaGetLastError());
}
void launch_move_rows(const float* svecs, const long long* sids, const float* snorms, const long long* src_rows,
                      const long long* dst_rows, int64_t n, int d, float* dvecs, long long* dids, float* dnorms,
                      cudaStream_t s) {
  if (n <= 0) return;
  move_rows_kernel<<<(unsigned)cdiv(n * 32, 256), 256, 0, s>>>(svecs, sids, snorms, src_rows, dst_rows, n, d, dvecs, dids, dnorms);
  B200VS_CUDA(cudaGetLastError());
}
void launch_set_ids(long long* ids, const long long* slots, int64_t n, long long value, cudaStream_t s) {
  if (n <= 0) return;
  set_ids_kernel<<<(unsigned)cdiv(n, 256), 256, 0, s>>>(ids, slots, n, value);
  B200VS_CUDA(cudaGetLastError());
}
static __global__ void negate_kernel(float* p, long long n) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) p[i] = -p[i];
}
void launch_negate(float* p, int64_t n, cudaStream_t s) {
  if (n > 0) negate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(p, n);
}

// VectorCalcDistance (src/vector/vector_index_utils.cc:48-124): one quad per (left, right) pair, reference order.
// Consecutive quads share the left row and walk the right rows, so a CTA re-reads a handful of rows from L1/L2.
// Dist is the exact scan's per-row functor (scan_kernels.cuh): Fp32Dist<L2> on float rows (d floats), HammingDist on
// zero-padded binary rows (d 32-bit words).
template <class Dist>
static __global__ void __launch_bounds__(256) pair_distance_kernel(const float* __restrict__ a, long long nl, const float* __restrict__ b,
                                                                   long long nr, int d, float* __restrict__ out) {
  const long long pair = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
  const int t = threadIdx.x & 3;
  const long long total = nl * nr;
  const bool valid = pair < total;
  const long long p = valid ? pair : 0;
  const long long i = p / nr, j = p % nr;
  const float v = Dist::eval(a, i, b + (size_t)j * d, d, t, (d & 3) == 0);
  if (valid && t == 0) out[p] = Dist::kL2 ? v : __fsub_rn(1.0f, v);
}
template <class Dist>
static void launch_pair(const float* a, int64_t nl, const float* b, int64_t nr, int d, float* out, cudaStream_t s) {
  const int64_t total = nl * nr;
  if (total <= 0) return;
  const unsigned grid = (unsigned)((total * 4 + 255) / 256);
  pair_distance_kernel<Dist><<<grid, 256, 0, s>>>(a, nl, b, nr, d, out);
  B200VS_CUDA(cudaGetLastError());
}
void launch_pair_distance(bool l2, const float* a, int64_t nl, const float* b, int64_t nr, int d, float* out, cudaStream_t s) {
  if (l2) launch_pair<Fp32Dist<true>>(a, nl, b, nr, d, out, s);
  else launch_pair<Fp32Dist<false>>(a, nl, b, nr, d, out, s);
}
void launch_pair_hamming(const uint32_t* a, int64_t nl, const uint32_t* b, int64_t nr, int w, float* out, cudaStream_t s) {
  launch_pair<HammingDist>(reinterpret_cast<const float*>(a), nl, reinterpret_cast<const float*>(b), nr, w, out, s);
}

void launch_iota(long long* p, int64_t n, cudaStream_t s) {
  if (n <= 0) return;
  iota_kernel<<<(unsigned)cdiv(n, 256), 256, 0, s>>>(p, n);
  B200VS_CUDA(cudaGetLastError());
}
// k-means centroid update: sums[assign[i]] += x[i], counts[assign[i]] += 1 (float atomics; order-free)
__global__ void kmeans_accumulate_kernel(const float* __restrict__ x, const long long* __restrict__ assign, long long n,
                                         int d, double scale, long long* sums, int* counts) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const long long c = assign[w];
  if (c < 0) return;
  const float* row = x + (size_t)w * d;
  unsigned long long* dst = reinterpret_cast<unsigned long long*>(sums + (size_t)c * d);
  for (int i = lane; i < d; i += 32) atomicAdd(dst + i, (unsigned long long)__double2ll_rn((double)row[i] * scale));
  if (lane == 0) atomicAdd(counts + c, 1);
}
void launch_kmeans_accumulate(const float* x, const long long* assign, int64_t n, int d, double scale, long long* sums,
                              int* counts, cudaStream_t s) {
  if (n <= 0) return;
  kmeans_accumulate_kernel<<<(unsigned)cdiv(n * 32, 256), 256, 0, s>>>(x, assign, n, d, scale, sums, counts);
  B200VS_CUDA(cudaGetLastError());
}

void launch_merge_api(int nparts, int64_t nq, int k, const float* pd, const long long* pi, float* od, long long* oi,
                      cudaStream_t s) {
  if (nq <= 0 || k <= 0) return;
  const int cap = select_pool_cap(k, SCAN_THREADS);
  const size_t smem = BlockSelect::smem_bytes(cap);
  ensure_smem(merge_api_kernel, smem);
  merge_api_kernel<<<(unsigned)nq, SCAN_THREADS, smem, s>>>(pd, pi, nparts, nq, k, cap, od, oi);
  B200VS_CUDA(cudaGetLastError());
}

}  // namespace b200vs
