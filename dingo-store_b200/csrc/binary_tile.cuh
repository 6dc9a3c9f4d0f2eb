// binary_tile.cuh — batched Hamming search of Binary Flat / Binary IVF-Flat on a list-major BMMA tile scan (binary_tile.cu).
#pragma once
#include "tc_scan.cuh"

namespace b200vs {

// true when a binary search takes the tile scan (otherwise the caller runs the exact Hamming scan).  v: the index's rows as
// lists (v.vecs = the packed words, v.ids, list layout and chunk counts; no norms).  cand: expected candidate rows per
// query (Flat: the rows; IVF: rows x nprobe / nlist), which decides with nq and k which path is faster.
bool bt_eligible(const TcView& v, int64_t nq, int k, int nprobe, double cand, const SearchCtx& sc);

// q: device queries [nq, w] (w = 32-bit words per row, zero padded).  probes: device [nq, nprobe] list indices (Flat: all
// zeros, nprobe = 1).  exact: the index's exact Hamming scan for the same probes and filter (exact.sc), which re-runs the
// queries the tile scan cannot answer.  Results equal the exact scan's, ids and distances.
void bt_search(IndexBase* ix, const TcView& v, int w, int64_t nq, const uint32_t* q, int k, const long long* probes, int nprobe,
               const ScanJob& exact, float* out_dist, long long* out_ids, cudaStream_t s);

}  // namespace b200vs
