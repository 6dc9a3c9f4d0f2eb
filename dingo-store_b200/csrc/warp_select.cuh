// warp_select.cuh — selection primitives of the per-query finish kernels (threshold, window select, coarse probe selection,
// tiny-batch top-k): the GPU form of the per-query heaps of the reference path (faiss HeapBlockResultHandler behind
// IndexIVF::search, src/vector/vector_index_ivf_flat.cc:247-251).
//
// Two forms of the same range-normalised radix select:
//   warp_kth_key       one warp, shuffles / ballots + a warp-private histogram, no block barrier.  Right when the keys sit in
//                      the warp's registers or a small staged array (<= ~1024 keys: threshold and coarse kernels).
//   block_kth_key_any  all threads of the CTA feed one shared histogram.  Right as soon as a CTA owns the query anyway: a lone
//                      warp executes dependent selection code at ~25 ns per instruction (nothing hides its latencies).
// Each kernel uses the form that measured faster (DESIGN.md 4.2).
#pragma once
#include "common.cuh"

namespace b200vs {

constexpr int WS_BINS = 512;  // histogram bins per narrowing step (9 bits), warp-private

// k-th smallest (k >= 1; at least k keys are visited) of the keys the warp's lanes enumerate through `for_each`
// (for_each(f) calls f(key) once per live key of THIS lane).  Range-normalised radix select: bin = (key - lo) >> shift
// over the live range [lo, hi], narrow to the bin that holds the k-th key, repeat until bins are one key wide.
// c_le = number of keys <= the result when it is known exactly, else k + 1.  All 32 lanes call; `hist` is a
// warp-private int[WS_BINS].
template <class ForEach>
__device__ __forceinline__ uint32_t warp_kth_key(int k, int* hist, ForEach for_each, int& c_le) {
  const int lane = threadIdx.x & 31;
  uint32_t mn = 0xFFFFFFFFu, mx = 0u;
  for_each([&](uint32_t key) { mn = min(mn, key); mx = max(mx, key); });
  uint32_t lo = __reduce_min_sync(0xffffffffu, mn), hi = __reduce_max_sync(0xffffffffu, mx);
  int kk = k;
  c_le = k + 1;
  for (;;) {
    const uint32_t range = hi - lo;
    if (range == 0) return lo;  // every remaining key is equal
    const int bits = 32 - __clz(range);
    const int shift = max(0, bits - 9);
    for (int i = lane; i < WS_BINS; i += 32) hist[i] = 0;
    __syncwarp();
    for_each([&](uint32_t key) { if (key >= lo && key <= hi) atomicAdd(&hist[(key - lo) >> shift], 1); });
    __syncwarp();
    constexpr int PER = WS_BINS / 32;
    int loc[PER], sum = 0;
#pragma unroll
    for (int j = 0; j < PER; ++j) { loc[j] = hist[lane * PER + j]; sum += loc[j]; }
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    const int before = incl - sum;
    const bool mine = before < kk && kk <= incl;  // exactly one lane
    int bin = 0, nk = 0, cle = 0;
    if (mine) {
      int acc = before;
#pragma unroll
      for (int j = 0; j < PER; ++j) {
        if (acc < kk && kk <= acc + loc[j]) { bin = lane * PER + j; nk = kk - acc; cle = (k - kk) + acc + loc[j]; }
        acc += loc[j];
      }
    }
    const int src = __ffs(__ballot_sync(0xffffffffu, mine)) - 1;
    bin = __shfl_sync(0xffffffffu, bin, src);
    nk = __shfl_sync(0xffffffffu, nk, src);
    cle = __shfl_sync(0xffffffffu, cle, src);
    const uint32_t nlo = lo + ((uint32_t)bin << shift);
    hi = min(hi, nlo + ((1u << shift) - 1u));
    lo = nlo;
    kk = nk;
    __syncwarp();
    if (shift == 0) { c_le = cle; return lo; }
  }
}

// ---------------------------------------------------------------------------------------------
// Block-cooperative form: ALL threads of the CTA take part.  A lone warp executes a selection at one instruction per
// ~25 ns (nothing hides its latencies: measured 8 us for 338 keys, 25 us for 2960), so whenever a CTA owns a query the
// whole CTA selects: every thread feeds its keys into one shared histogram, warp 0 locates the bin, two or three rounds.
// for_each(f) calls f(key) once per live key of THIS thread.  Returns the k-th smallest key to every thread; S.c_le as in
// warp_kth_key.  Barriers inside: every thread of the CTA must call.
// ---------------------------------------------------------------------------------------------
constexpr int BS_BINS = 1024;
struct BlockSelShared {
  int hist[BS_BINS];
  uint32_t red[2][32];
  uint32_t lo, hi;
  int k, c_le;
};
template <class ForEach>
__device__ __forceinline__ uint32_t block_kth_key_any(int k, BlockSelShared& S, ForEach for_each) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
  uint32_t mn = 0xFFFFFFFFu, mx = 0u;
  for_each([&](uint32_t key) { mn = min(mn, key); mx = max(mx, key); });
  mn = __reduce_min_sync(0xffffffffu, mn);
  mx = __reduce_max_sync(0xffffffffu, mx);
  if (lane == 0) { S.red[0][warp] = mn; S.red[1][warp] = mx; }
  __syncthreads();
  if (threadIdx.x < 32) {
    uint32_t a = lane < nwarps ? S.red[0][lane] : 0xFFFFFFFFu, b = lane < nwarps ? S.red[1][lane] : 0u;
    a = __reduce_min_sync(0xffffffffu, a);
    b = __reduce_max_sync(0xffffffffu, b);
    if (lane == 0) { S.lo = a; S.hi = b; S.k = k; S.c_le = k + 1; }
  }
  __syncthreads();
  for (;;) {
    const uint32_t lo = S.lo, hi = S.hi;
    const int kk = S.k;
    const uint32_t range = hi - lo;
    if (range == 0) return lo;  // every remaining key is equal
    const int bits = 32 - __clz(range);
    const int shift = max(0, bits - 10);
    for (int i = threadIdx.x; i < BS_BINS; i += blockDim.x) S.hist[i] = 0;
    __syncthreads();
    for_each([&](uint32_t key) { if (key >= lo && key <= hi) atomicAdd(&S.hist[(key - lo) >> shift], 1); });
    __syncthreads();
    if (threadIdx.x < 32) {  // locate the bin that holds the kk-th key: 32 bins per lane
      constexpr int PER = BS_BINS / 32;
      int sum = 0;
      for (int j = 0; j < PER; ++j) sum += S.hist[lane * PER + j];
      int incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
      const int before = incl - sum;
      if (before < kk && kk <= incl) {  // exactly one lane
        int acc = before;
        for (int j = 0; j < PER; ++j) {
          const int c = S.hist[lane * PER + j];
          if (acc < kk && kk <= acc + c) {
            const uint32_t nlo = lo + ((uint32_t)(lane * PER + j) << shift);
            S.lo = nlo;
            S.hi = min(hi, nlo + ((1u << shift) - 1u));
            S.k = kk - acc;
            if (shift == 0) S.c_le = (k - kk) + acc + c;
            break;
          }
          acc += c;
        }
      }
    }
    __syncthreads();
    if (shift == 0) return S.lo;
  }
}

// Rank sort of m (key, id) pairs in shared memory by all threads of the CTA: emit(rank, index) for every entry.
template <class Emit>
__device__ __forceinline__ void block_rank_sort(const uint32_t* kd, const long long* kid, int m, Emit emit) {
  for (int e = threadIdx.x; e < m; e += blockDim.x) {
    const uint32_t d0 = kd[e];
    const long long i0 = kid[e];
    int rank = 0;
    for (int j = 0; j < m; ++j) {
      const uint32_t dj = kd[j];
      const long long ij = kid[j];
      rank += (key_less(dj, ij, d0, i0) || (dj == d0 && ij == i0 && j < e)) ? 1 : 0;
    }
    emit(rank, e);
  }
}

}  // namespace b200vs
