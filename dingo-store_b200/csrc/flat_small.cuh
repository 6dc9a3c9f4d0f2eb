// flat_small.cuh — single-launch exact Flat search for tiny batches (see flat_small.cu).
#pragma once
#include "index.h"

namespace b200vs {

bool flat_small_eligible(int device, int64_t nq, int64_t n, int d, int k, const SearchCtx& sc);
// q: prepared queries (normalised for cosine), device; writes API-semantics results [nq, k], or the raw metric value
// (L2 distance | ip) when raw_out
void flat_small_search(IndexBase* ix, bool l2, const float* vecs, const long long* ids, int64_t n, int64_t nq, const float* q, int k,
                       const SearchCtx& sc, float* out_dist, long long* out_ids, bool raw_out, cudaStream_t s);

}  // namespace b200vs
