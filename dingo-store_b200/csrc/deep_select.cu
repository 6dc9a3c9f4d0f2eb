// deep_select.cu — exact top-k for k up to kDeepMaxK (b200vs_search_deep): the select stages after the key pass.
//
// Per query chunk: the key pass (the exact scan with DeepKeySink, launched by the caller) writes every candidate's key and
// eligibility; then
//   1. radix select of the k-th smallest eligible key T over 8-bit digits (4 histogram + pick passes, global histograms per
//      query), leaving the number of keys == T still needed;
//   2. only where more candidates tie at T than are needed: radix select of the needed smallest ids among them (8 passes over
//      the 64-bit ids), so ties resolve to the smallest ids as the (key, id) order of the shared-memory select does;
//   3. compaction of the <= k survivors into [nqc, k] (key, id) slots;
//   4. ordering by (key, id): a stable segmented sort by id, then a stable one by key (CUB, off the scan);
//   5. the key -> API distance conversion of merge_select_kernel, and -1 / 0 padding.
#include <cub/device/device_segmented_sort.cuh>

#include <algorithm>

#include "index.h"

namespace b200vs {

namespace {

constexpr int DT = 256;                         // threads of the select kernels
constexpr long long kDeepBudget = 1LL << 30;    // bytes of one query chunk's key space and survivor buffers

// the select state of one query
struct DeepState {
  uint32_t key;             // the key prefix found so far, then T
  int mode;                 // 0: every eligible candidate survives; 1: keys < T and every key == T; 2: keys < T, and keys == T
                            //    with id < the id threshold or (id == it, up to `need` of them)
  long long need;           // rank still to find inside the current prefix; after the selects, the == threshold survivors
  unsigned long long id;    // the id prefix (mode 2), then the id threshold
  unsigned long long cnt;   // candidates inside the prefix chosen by the last pick
  unsigned long long taken; // id == threshold survivors handed out (compaction)
  unsigned long long out;   // survivors written (compaction)
};

// candidate position -> row of the index, with the exact scan's map_row rule; q is chunk-local
struct Space {
  int mode;
  long long n, row_stride;
  const long long* ids;       // chunk-relative on a dense space with row_stride
  const long long* probes;    // chunk-relative [nqc, nprobe]
  int nprobe;
  const long long* list_off;
  const long long* pre;       // chunk-relative [nqc, nprobe + 1]
  __device__ long long total(int q) const { return mode == 0 ? n : pre[(size_t)q * (nprobe + 1) + nprobe]; }
  __device__ long long id(int q, long long i) const {
    if (mode == 0) return ids[(size_t)q * row_stride + i];
    const long long* pq = pre + (size_t)q * (nprobe + 1);
    int lo = 0, hi = nprobe - 1;  // last p with pq[p] <= i
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (pq[mid] <= i) lo = mid; else hi = mid - 1;
    }
    return ids[list_off[probes[(size_t)q * nprobe + lo]] + (i - pq[lo])];
  }
};

// this block's share [c0, c1) of query q's candidates, whole multiples of DT so every warp runs the same iterations
__device__ __forceinline__ void block_range(long long total, long long& c0, long long& c1) {
  const long long per = cdiv(cdiv(total, gridDim.x), DT) * DT;
  c0 = (long long)blockIdx.x * per;
  c1 = std::min(total, c0 + per);
}

// probe-prefix positions of a list space: pre[q][p] = rows of probes 0 .. p-1, pre[q][nprobe] = the query's candidates; *cmax
// = the largest of those.  One warp per query.
__global__ void deep_prefix_kernel(const long long* probes, const int* list_len, long long nq, int nprobe, long long* pre,
                                   unsigned long long* cmax) {
  const long long q = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (q >= nq) return;
  long long carry = 0;
  for (int base = 0; base < nprobe; base += 32) {
    const int p = base + lane;
    long long len = 0;
    if (p < nprobe) { const long long l = probes[(size_t)q * nprobe + p]; len = l >= 0 ? list_len[l] : 0; }
    long long incl = len;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const long long v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    if (p < nprobe) pre[(size_t)q * (nprobe + 1) + p] = carry + incl - len;
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (lane == 0) {
    pre[(size_t)q * (nprobe + 1) + nprobe] = carry;
    atomicMax(cmax, (unsigned long long)carry);
  }
}

__global__ void deep_init_kernel(const unsigned long long* count, int nqc, int k, DeepState* st) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nqc) return;
  DeepState s{};
  s.mode = count[q] > (unsigned long long)k ? 1 : 0;
  s.need = k;
  st[q] = s;
}

// one digit pass: hist[q][digit] over the candidates inside the current prefix.  IDS: the ids of the keys == T (mode 2 only);
// otherwise the keys (mode 1 only).  Grid (bx, nqc).
template <bool IDS>
__global__ void __launch_bounds__(DT) deep_hist_kernel(const Space sp, const uint32_t* keys, const unsigned char* elig, long long stride,
                                                       const DeepState* st, int shift, unsigned long long* hist) {
  const int q = blockIdx.y;
  const DeepState s = st[q];
  if (s.mode != (IDS ? 2 : 1)) return;
  __shared__ unsigned int h[256];
  for (int i = threadIdx.x; i < 256; i += DT) h[i] = 0;
  __syncthreads();
  long long c0, c1;
  block_range(sp.total(q), c0, c1);
  const uint32_t* kq = keys + (size_t)q * stride;
  const unsigned char* eq = elig + (size_t)q * stride;
  const bool top = shift + 8 >= (IDS ? 64 : 32);
  const int lane = threadIdx.x & 31;
  for (long long base = c0; base < c1; base += DT) {  // whole warps per step: the digit's peers add once per warp
    const long long i = base + threadIdx.x;
    int digit = -1;
    if (i < c1 && eq[i]) {
      const uint32_t key = kq[i];
      if (IDS) {
        if (key == s.key) {
          const unsigned long long id = (unsigned long long)sp.id(q, i);
          if (top || ((id ^ s.id) >> (shift + 8)) == 0) digit = (int)((id >> shift) & 255);
        }
      } else if (top || (((unsigned long long)(key ^ s.key)) >> (shift + 8)) == 0) {
        digit = (int)((key >> shift) & 255);
      }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, digit);
    if (digit >= 0 && lane == __ffs(peers) - 1) atomicAdd(&h[digit], (unsigned)__popc(peers));
  }
  __syncthreads();
  for (int b = threadIdx.x; b < 256; b += DT)
    if (h[b]) atomicAdd(&hist[(size_t)q * 256 + b], (unsigned long long)h[b]);
}

// the digit holding rank `need` of the current prefix: prefix |= digit << shift, need -= the candidates below it.  Clears the
// histogram for the next pass.  One block of 256 threads per query.
template <bool IDS>
__global__ void __launch_bounds__(256) deep_pick_kernel(DeepState* st, int shift, unsigned long long* hist) {
  const int q = blockIdx.x, b = threadIdx.x, lane = b & 31, warp = b >> 5;
  __shared__ unsigned long long wsum[8];
  const bool active = st[q].mode == (IDS ? 2 : 1);
  const unsigned long long need = (unsigned long long)st[q].need;  // read by every thread before the one winner writes
  unsigned long long* hq = hist + (size_t)q * 256;
  const unsigned long long c = hq[b];
  hq[b] = 0;
  if (!active) return;  // block-uniform
  unsigned long long incl = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  for (int w = 0; w < warp; ++w) incl += wsum[w];
  const unsigned long long excl = incl - c;
  DeepState& s = st[q];
  if (c > 0 && excl < need && need <= incl) {
    if (IDS) s.id |= (unsigned long long)b << shift;
    else s.key |= (uint32_t)b << shift;
    s.need = (long long)(need - excl);
    s.cnt = c;
    if (!IDS && shift == 0 && c > need - excl) s.mode = 2;  // more keys == T than survivors: resolve them by id
  }
}

// survivors -> [q][0, out) of okey / oid, in no particular order.  Grid (bx, nqc).
__global__ void __launch_bounds__(DT) deep_compact_kernel(const Space sp, const uint32_t* keys, const unsigned char* elig, long long stride,
                                                          DeepState* st, int k, uint32_t* okey, long long* oid) {
  const int q = blockIdx.y, lane = threadIdx.x & 31;
  const DeepState s = st[q];
  long long c0, c1;
  block_range(sp.total(q), c0, c1);
  const uint32_t* kq = keys + (size_t)q * stride;
  const unsigned char* eq = elig + (size_t)q * stride;
  for (long long base = c0; base < c1; base += DT) {
    const long long i = base + threadIdx.x;
    bool take = false;
    uint32_t key = 0;
    long long id = -1;
    if (i < c1 && eq[i]) {
      key = kq[i];
      if (s.mode == 0 || key < s.key) {
        take = true;
      } else if (key == s.key) {
        if (s.mode == 1) {
          take = true;
        } else {
          id = sp.id(q, i);
          const unsigned long long u = (unsigned long long)id;
          take = u < s.id || (u == s.id && atomicAdd(&st[q].taken, 1ULL) < (unsigned long long)s.need);
        }
      }
      if (take && id < 0) id = sp.id(q, i);
    }
    const unsigned m = __ballot_sync(0xffffffffu, take);
    if (!m) continue;
    unsigned long long slot0 = 0;
    const int leader = __ffs(m) - 1;
    if (lane == leader) slot0 = atomicAdd(&st[q].out, (unsigned long long)__popc(m));
    slot0 = __shfl_sync(0xffffffffu, slot0, leader);
    if (take) {
      const size_t o = (size_t)q * k + slot0 + __popc(m & ((1u << lane) - 1u));
      okey[o] = key;
      oid[o] = id;
    }
  }
}

__global__ void deep_offsets_kernel(const DeepState* st, int nqc, int k, int* begin, int* end) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nqc) return;
  begin[q] = q * k;
  end[q] = q * k + (int)st[q].out;
}

// sorted survivors -> results of queries q0 + [0, nqc): merge_select_kernel's conversion (raw: the metric value; otherwise
// the API distance), or the key's own float when the keys are API distances; -1 / 0 past the survivors
__global__ void deep_emit_kernel(const uint32_t* okey, const long long* oid, const DeepState* st, int k, bool l2, bool api_keys, bool raw,
                                 long long q0, float* od, long long* oi) {
  const int q = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k) return;
  const long long have = (long long)st[q].out;
  float dv = 0.f;
  long long id = -1;
  if (i < have) {
    const float v = ord2f(okey[(size_t)q * k + i]);
    if (api_keys) {
      dv = v;
    } else {
      const float rv = l2 ? v : -v;
      dv = raw ? rv : (l2 ? rv : __fsub_rn(1.0f, rv));  // FillSearchResult, vector_index_utils.cc:632-634
    }
    id = oid[(size_t)q * k + i];
  }
  if (od) od[(size_t)(q0 + q) * k + i] = dv;
  oi[(size_t)(q0 + q) * k + i] = id;
}

// key pass of a merge of API-distance lists [nqc, n] (running result + tile of the brute-force scan): key f2ord(distance), as
// merge_api_kernel ranks them; a slot is eligible when it holds an id.  Grid (cdiv(n, 256), nqc).
__global__ void deep_api_keys_kernel(const float* d, const long long* ids, long long n, DeepKeys o) {
  const int q = blockIdx.y;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool ok = i < n && ids[(size_t)q * n + i] >= 0;
  if (ok) {
    o.keys[(size_t)q * o.stride + i] = f2ord(d[(size_t)q * n + i]);
    o.elig[(size_t)q * o.stride + i] = 1;
  }
  const unsigned c = __popc(__ballot_sync(0xffffffffu, ok));
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(o.count + q, (unsigned long long)c);
}

// bump allocation from one device buffer (256-byte aligned pieces)
struct Carve {
  unsigned char* p;
  size_t used = 0;
  template <class T>
  T* take(size_t n) {
    T* r = reinterpret_cast<T*>(p + used);
    used += (n * sizeof(T) + 255) / 256 * 256;
    return r;
  }
  template <class T>
  static size_t bytes(size_t n) { return (n * sizeof(T) + 255) / 256 * 256; }
};

}  // namespace

void run_deep_merge_api(IndexBase* ix, int64_t nq, int k, int n, const float* cat_d, const long long* cat_i, float* od, long long* oi,
                        cudaStream_t s) {
  DeepJob dj;
  dj.api_keys = true; dj.mode = 0; dj.n = n; dj.row_stride = n; dj.ids = cat_i;
  run_deep(ix, dj, nq, k, od, false, oi, [&](int64_t q0, int nqc, const DeepKeys& o, cudaStream_t st) {
    deep_api_keys_kernel<<<dim3((unsigned)cdiv(n, 256), (unsigned)nqc), 256, 0, st>>>(cat_d + (size_t)q0 * n, cat_i + (size_t)q0 * n, n, o);
    B200VS_CUDA(cudaGetLastError());
    ix->launch_count(1);
  }, s);
}

void run_deep(IndexBase* ix, const DeepJob& job, int64_t nq, int k, float* od, bool raw, long long* oi, const DeepKeyPass& pass,
              cudaStream_t s) {
  if (nq <= 0 || k <= 0) return;
  if (k > kDeepMaxK) fail(B200VS_EILLEGAL_PARAMETERS, "topk above " + std::to_string(kDeepMaxK));
  // the candidate space: rows [0, n), or the probe-prefix positions of every query (one device-to-host read of the largest)
  long long cmax = job.n;
  long long* pre = nullptr;
  if (job.mode == 1) {
    pre = ix->scratch.alloc<long long>((size_t)nq * (job.nprobe + 1));
    unsigned long long* dmax = ix->scratch.alloc<unsigned long long>(1);
    B200VS_CUDA(cudaMemsetAsync(dmax, 0, 8, s));
    deep_prefix_kernel<<<(unsigned)cdiv(nq * 32, 256), 256, 0, s>>>(job.probes, job.list_len, nq, job.nprobe, pre, dmax);
    B200VS_CUDA(cudaGetLastError());
    unsigned long long h = 0;
    B200VS_CUDA(cudaMemcpyAsync(&h, dmax, 8, cudaMemcpyDeviceToHost, s));
    B200VS_CUDA(cudaStreamSynchronize(s));
    cmax = (long long)h;
    ix->launch_count(1);
  }
  // queries per chunk: keys + eligibility (5 B per candidate) and the survivor buffers (24 B per slot) within the budget
  const long long per_query = cmax * 5 + (long long)k * 24 + 4096;
  int64_t nqc_max = std::max<int64_t>(1, std::min<int64_t>({nq, kDeepBudget / per_query, 65535, INT32_MAX / k}));
  // the chunk's buffers: one stream-ordered allocation for this call, freed stream-ordered when it returns (no device-wide
  // synchronisation, nothing kept in the lane's scratch); a device short of memory gets smaller chunks, down to one query
  size_t sort_bytes = 0, total = 0;
  auto sizes = [&](int64_t m) {
    const size_t slots = (size_t)m * k, space = (size_t)m * cmax;
    size_t tb = 0;
    sort_bytes = 0;
    B200VS_CUDA(cub::DeviceSegmentedSort::StableSortPairs(nullptr, tb, (const long long*)nullptr, (long long*)nullptr, (const uint32_t*)nullptr,
                                                          (uint32_t*)nullptr, (int)slots, (int)m, (int*)nullptr, (int*)nullptr, s));
    sort_bytes = std::max(sort_bytes, tb);
    B200VS_CUDA(cub::DeviceSegmentedSort::StableSortPairs(nullptr, tb, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const long long*)nullptr,
                                                          (long long*)nullptr, (int)slots, (int)m, (int*)nullptr, (int*)nullptr, s));
    sort_bytes = std::max(sort_bytes, tb);
    total = Carve::bytes<uint32_t>(space) + Carve::bytes<unsigned char>(space) + Carve::bytes<unsigned long long>(m) +
            Carve::bytes<DeepState>(m) + Carve::bytes<unsigned long long>((size_t)m * 256) + 2 * Carve::bytes<uint32_t>(slots) +
            2 * Carve::bytes<long long>(slots) + 2 * Carve::bytes<int>(m) + Carve::bytes<unsigned char>(sort_bytes);
  };
  struct StreamBuf {
    void* p = nullptr;
    cudaStream_t s;
    ~StreamBuf() { if (p) cudaFreeAsync(p, s); }
  } buf{nullptr, s};
  for (;;) {
    sizes(nqc_max);
    const cudaError_t e = cudaMallocAsync(&buf.p, total, s);
    if (e == cudaSuccess) break;
    if (e != cudaErrorMemoryAllocation || nqc_max == 1) B200VS_CUDA(e);
    cudaGetLastError();  // clear the failed allocation
    buf.p = nullptr;
    nqc_max = (nqc_max + 1) / 2;
  }
  const size_t slots = (size_t)nqc_max * k, space = (size_t)nqc_max * cmax;
  Carve c{static_cast<unsigned char*>(buf.p)};
  DeepKeys o;
  o.keys = c.take<uint32_t>(space);
  o.elig = c.take<unsigned char>(space);
  o.count = c.take<unsigned long long>(nqc_max);
  o.stride = cmax;
  o.nprobe = job.nprobe;
  DeepState* st = c.take<DeepState>(nqc_max);
  unsigned long long* hist = c.take<unsigned long long>((size_t)nqc_max * 256);
  uint32_t* okey = c.take<uint32_t>(slots);
  uint32_t* skey = c.take<uint32_t>(slots);
  long long* oid = c.take<long long>(slots);
  long long* sid = c.take<long long>(slots);
  int* d_begin = c.take<int>(nqc_max);
  int* d_end = c.take<int>(nqc_max);
  void* sort_tmp = c.take<unsigned char>(sort_bytes);
  size_t tb = 0;
  B200VS_CUDA(cudaMemsetAsync(hist, 0, (size_t)nqc_max * 256 * 8, s));  // each pick clears what it read

  const int sms = device_sm_count(ix->device);
  for (int64_t q0 = 0; q0 < nq; q0 += nqc_max) {
    const int nqc = (int)std::min<int64_t>(nqc_max, nq - q0);
    B200VS_CUDA(cudaMemsetAsync(o.elig, 0, (size_t)nqc * cmax, s));
    B200VS_CUDA(cudaMemsetAsync(o.count, 0, (size_t)nqc * 8, s));
    o.pre = pre ? pre + (size_t)q0 * (job.nprobe + 1) : nullptr;
    if (cmax > 0) pass(q0, nqc, o, s);

    Space sp;
    sp.mode = job.mode; sp.n = job.n; sp.row_stride = job.row_stride; sp.nprobe = job.nprobe; sp.list_off = job.list_off; sp.pre = o.pre;
    sp.ids = job.mode == 0 ? job.ids + (size_t)q0 * job.row_stride : job.ids;
    sp.probes = job.probes ? job.probes + (size_t)q0 * job.nprobe : nullptr;
    const unsigned bx = (unsigned)std::max<int64_t>(1, std::min<int64_t>(cdiv(std::max(cmax, 1LL), 16384), std::max(1, sms * 8 / nqc)));
    const dim3 grid(bx, (unsigned)nqc);
    deep_init_kernel<<<(unsigned)cdiv(nqc, 256), 256, 0, s>>>(o.count, nqc, k, st);
    for (int shift = 24; shift >= 0; shift -= 8) {
      deep_hist_kernel<false><<<grid, DT, 0, s>>>(sp, o.keys, o.elig, cmax, st, shift, hist);
      deep_pick_kernel<false><<<(unsigned)nqc, 256, 0, s>>>(st, shift, hist);
    }
    for (int shift = 56; shift >= 0; shift -= 8) {  // blocks of queries without a tie to resolve return at once
      deep_hist_kernel<true><<<grid, DT, 0, s>>>(sp, o.keys, o.elig, cmax, st, shift, hist);
      deep_pick_kernel<true><<<(unsigned)nqc, 256, 0, s>>>(st, shift, hist);
    }
    deep_compact_kernel<<<grid, DT, 0, s>>>(sp, o.keys, o.elig, cmax, st, k, okey, oid);
    deep_offsets_kernel<<<(unsigned)cdiv(nqc, 256), 256, 0, s>>>(st, nqc, k, d_begin, d_end);
    B200VS_CUDA(cudaGetLastError());
    // (key, id) order: stable by id, then stable by key
    tb = sort_bytes;
    B200VS_CUDA(cub::DeviceSegmentedSort::StableSortPairs(sort_tmp, tb, oid, sid, okey, skey, nqc * k, nqc, d_begin, d_end, s));
    tb = sort_bytes;
    B200VS_CUDA(cub::DeviceSegmentedSort::StableSortPairs(sort_tmp, tb, skey, okey, sid, oid, nqc * k, nqc, d_begin, d_end, s));
    deep_emit_kernel<<<dim3((unsigned)cdiv(k, 256), (unsigned)nqc), 256, 0, s>>>(okey, oid, st, k, job.l2, job.api_keys, raw, q0, od, oi);
    B200VS_CUDA(cudaGetLastError());
    ix->launch_count(1 + 2 * 4 + 2 * 8 + 2 + 2 + 1);
  }
}

}  // namespace b200vs
