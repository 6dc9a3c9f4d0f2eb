// tc_scan.cuh — tensor-core candidate pass for Flat / IVF-Flat search (sm_90a: TMA + wgmma + mbarrier).
//
// What it replaces: the per-query CPU scans IVFFlatScanner::scan_codes / exhaustive_*_seq behind
// VectorIndexIvfFlat::Search and VectorIndexFlat::Search (src/vector/vector_index_ivf_flat.cc:247-251,
// vector_index_flat.cc:249-252) and the IndexFlat coarse quantiser of IVF (vector_index_ivf_flat.cc:805-837).
// The reference streams every probed list once PER QUERY on one core; here each probed list chunk is streamed
// from HBM ONCE PER BATCH and multiplied against all queries that probe it — the one place on this path where
// the work is a dense contraction (SURVEY.md §8d).
//
// Exactness: the MMA runs in TF32 (operands truncated to 10 mantissa bits) or, on an IVF-Flat index's FP16 mirror, in
// FP16 (rows and queries scaled by a power of two and rounded to nearest), so its scores only SELECT candidates.  Per query the engine keeps every row whose approximate score is within 2*eps of the k-th best
// approximate score (eps = rigorous bound on the TF32 score error); all of those are re-scored by the exact
// FP32 kernel in the reference's AVX-512 order, so the returned ids and distances are identical to the exact
// path.  Queries whose window cannot be certified (candidate overflow / threshold too tight) are re-run on
// the exact scan.  See DESIGN.md §Tensor-core candidate pass.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include "filter.cuh"
#include "index.h"

namespace b200vs {

constexpr int TC_BM = 128;        // database rows per tile (two warpgroups x wgmma M = 64)
constexpr int TC_BK = 32;         // floats per K block = 128 B = one swizzle span (64 halves on the FP16 path)
constexpr int TC_NQT = 128;       // queries per work item (wgmma N <= 128): a probed list chunk is re-streamed only beyond 128 queries
constexpr int TC_CHUNK = 512;     // rows per work item (list chunk): fine grain for dynamic load balance
constexpr int TC_SPAN = 2048;     // one sampled chunk per TC_SPAN rows of a list
constexpr int TC_HITS = 256;      // captured rows staged per consumer warp between flushes
constexpr int TC_SAMPLE = 32;     // sampled rows per span for the threshold estimate
constexpr int TC_SQ = 4;          // scheduler queue depth (items the producer may run ahead)
constexpr uint32_t TC_A_BYTES = TC_BM * 128;
constexpr uint32_t TC_B_BYTES = TC_NQT * 128;

struct TcItem {
  int list;
  int row_begin, row_end;  // rows within the list
  int pair_begin;          // first row of this item's query group in the gathered-query workspace
  int nq;                  // queries in the group (1..TC_NQT)
  int sample_slot;         // >= 0 when this item is a sampled chunk
  int pad[2];
};

struct TcParams {
  const long long* ids;
  const float* norms;
  const long long* list_off;
  int d;
  const TcItem* items;
  const int* totals;        // [0] n_items  [1] n_pairs  [2] n_sample_items
  const int* sample_list;   // [n_sample_items] item indices
  int* work_counter;        // dynamic scheduler: next work index
  const int* pair_query;    // [npairs] query index of each gathered row
  int mode;                 // 0 = sample pass, 1 = capture pass, 2 = dense pass (every score written)
  float* sample;            // mode 0: [sample_items, TC_NQT, TC_SAMPLE]
  const float* tau;         // mode 1: [nq] capture threshold on the approximate score
  unsigned long long* cand; // mode 1: [nq, cap]  (ord(score) << 32 | arena row)
  int* cand_cnt;            // mode 1: [nq]
  int cap;
  float* dense;             // mode 2: [nq, dense_ld] approximate scores (row = column index)
  long long dense_ld;
  int split;                // error-compensated TF32: hi*hi + lo*hi + hi*lo into one accumulator (coarse quantiser)
  const float* hscale;      // FP16 path: [arena rows] power-of-two scale of each row of the mirror
  const float* qscale;      // FP16 path: [nq] power-of-two scale of each query
  int l2;
  FilterDev filt;
};

// view of an index the tile scan can run on (lists contiguous in one arena)
struct TcView {
  const float* vecs = nullptr;
  const long long* ids = nullptr;
  const float* norms = nullptr;
  int64_t arena_rows = 0;               // rows addressable by the A tensor map
  const long long* list_off = nullptr;  // device [nlist]
  const int* list_len = nullptr;        // device [nlist]
  int nlist = 0;
  int64_t total_chunks = 0;  // sum over lists of ceil(len / TC_CHUNK)   (host bookkeeping)
  int max_chunks_per_list = 0;
  float max_norm = 0.f;      // max ||x|| over the index (host bookkeeping, monotone)
  const float* vecs_hi = nullptr;  // optional split of the rows for the error-compensated coarse pass:
  const float* vecs_lo = nullptr;  //   hi = x with the low 13 mantissa bits cleared, lo = x - hi (both exact)
  bool flat = false;         // single list covering rows [0, arena_rows)
  long long id_offset = 0;   // tc_coarse on a slice of the centroid table: added to the returned row indices
  bool api_scores = false;   // tc_coarse: return the ascending ranking score (L2 distance | -ip) instead of the raw metric value
  const __half* vecs_h = nullptr;  // optional FP16 mirror of vecs (x * 2^-e per row, rounded to nearest): the list scan
  const float* hscale = nullptr;   //   streams it instead of the FP32 rows; hscale[r] = 2^e (DESIGN.md 3, 4.2)
};

// The one-list layout of a Flat view over rows [0, rows): off_dev[0] = 0 and len_dev[0] = rows, on the device
inline void set_flat_layout(TcView& v, int64_t rows, const long long* off_dev, const int* len_dev) {
  v.arena_rows = rows; v.list_off = off_dev; v.list_len = len_dev;
  v.nlist = 1; v.flat = true; v.total_chunks = (rows + TC_CHUNK - 1) / TC_CHUNK; v.max_chunks_per_list = (int)v.total_chunks;
}

// Arithmetic of the tile kernel's scores, and so of the error bound tc_eps()
enum TcArith : int {
  TC_ARITH_TF32 = 0,   // rows truncated to TF32, queries rounded to nearest (list scan without a mirror)
  TC_ARITH_SPLIT = 1,  // error-compensated hi / lo TF32 (coarse quantiser)
  TC_ARITH_FP16 = 2,   // rows and queries scaled by powers of two and rounded to FP16 (list scan on the mirror)
};

// true when this search can use the tensor-core pass (otherwise the caller runs the exact scan).  Top-k: k <= 128.  Range
// (k = max_results): k <= 4096, the select's limit, and the streaming finish's shared memory fits.
bool tc_eligible(const IndexBase* ix, const TcView& v, int64_t nq, int k, int nprobe, const SearchCtx& sc, bool range);
// the plan-size half of tc_eligible: the view's rows, the (query, probe) pairs, work items and sample buffer fit the plan
bool tc_plan_fits(const TcView& v, int64_t nq, int nprobe);
// false when no query can have a finite error bound against rows of this max ||x|| (tc_eps), so the tile passes would
// only be thrown away: L2 with max ||x||^2 > 2^125, IP / cosine with max ||x|| not finite
bool tc_norms_in_range(bool l2, float max_norm);

// Probes -> (list, query) pairs -> work items, shared by the float and the binary tile scans.  Uses v.nlist, v.list_len
// and the chunk counts.  qrows: device query rows of row_bytes each (a multiple of 16), copied pair by pair into bws.
struct TcPairs {
  int *cnt, *pos, *pair_off, *item_off, *totals, *pair_query, *sample_list, *work;
  void* bws;  // [npairs + TC_NQT] gathered query rows: a work item's B block is nq <= TC_NQT consecutive rows
  TcItem* items;
  int64_t bound, sbound, npairs;  // host bounds on the work items and on the sampled items
};
TcPairs tc_plan_pairs(IndexBase* ix, const TcView& v, int64_t nq, const long long* probes, int nprobe, const void* qrows,
                      int row_bytes, cudaStream_t s);
int tc_cand_cap(int k);  // captured rows kept per query
// qmap[0, *count) = the queries whose flags[q] != 0, in no particular order
void tc_compact_flags(const int* flags, int nq, int* qmap, int* count, cudaStream_t s);
// exact re-run of the queries in qmap[0, *qcount) (kernels.cu)
void run_scan_mapped(IndexBase* ix, const ScanJob& job, int64_t nq_max, const int* qmap, const int* qcount, const float* queries,
                     int k, float* out_dist, float* out_raw, long long* out_ids, int* out_counts, cudaStream_t s);

// The tile scan of r over probes: device [nq, nprobe] list indices (for Flat: all zeros, nprobe = 1).  q: device queries,
// already normalised for cosine.  Top-k: the capture threshold of each query comes from a sample pass.  Range (r.range,
// thr_raw: L2 keeps dist < thr_raw, IP / cosine keep ip > thr_raw): it comes from the radius widened by tc_eps, and the
// closest r.k hits are kept by (distance, id), as the exact scan with the same threshold keeps them, with the count of
// each query in r.oc.  Every captured row is re-scored exactly; r.od holds API distances, or the raw metric value
// (L2 distance | ip) when r.raw.  Queries the tile passes cannot certify (or whose capture overflows) re-run on the exact scan.
void tc_search(IndexBase* ix, const TcView& v, const SearchReq& r, const float* q, const long long* probes, int nprobe, float thr_raw,
               cudaStream_t s);

// Exact top-nprobe of every query against a small row set (the IVF coarse quantiser): dense TF32 score matrix on the
// tensor cores, then window select + exact FP32 re-score.  Always certified (every score is available).
// out_probes [nq, nprobe] row indices; out_raw (optional) [nq, nprobe] raw metric values (L2 distance / ip).
bool tc_coarse_eligible(const IndexBase* ix, int64_t nq, int nrows, int nprobe);
void tc_coarse(IndexBase* ix, const TcView& v, bool l2, int64_t nq, const float* q, int nprobe, long long* out_probes,
               float* out_raw, cudaStream_t s);

// Diagnostics (b200vs_debug_tc_scores; no search path calls it): the tile kernel's dense approximate scores of q (device,
// prepared) against every arena row, out_scores [nq, v.arena_rows], and the tc_eps() the finish kernels use, out_eps [nq].
// arith: TC_ARITH_TF32 = list scan without a mirror, TC_ARITH_SPLIT = the coarse pass's hi / lo arithmetic,
// TC_ARITH_FP16 = list scan on an FP16 mirror (a temporary one is made from v.vecs inside the call).
// sample (v.flat, TC_ARITH_TF32 or TC_ARITH_FP16): the sample pass's scores instead, from the kernel's sample
// configuration, for the rows it samples (the first TC_SAMPLE rows of every TC_SPAN); every other row is NaN.
void tc_debug_scores(IndexBase* ix, const TcView& v, bool l2, int64_t nq, const float* q, TcArith arith, bool sample,
                     float* out_scores, float* out_eps, cudaStream_t s);

float device_max_norm(IndexBase* ix, const float* norms_sq, int64_t n, cudaStream_t s);  // sqrt(max ||x||^2)
void launch_row_norms(const float* x, int64_t n, int d, float* out, cudaStream_t s);     // out[i] = <x_i, x_i>
void launch_split_rows(const float* x, int64_t n, int d, float* hi, float* lo, cudaStream_t s);
// FP16 mirror rows: for i < n, row r = rows ? rows[i] : i, half[r] = RN(x[r] * 2^-e), scale[r] = 2^e with
// max |x[r]| * 2^-e in [2^14, 2^15) (a zero row: scale 1).  d % 8 == 0.
void launch_half_rows(const float* x, const long long* rows, int64_t n, int d, __half* half, float* scale, cudaStream_t s);

}  // namespace b200vs
