// binary_tile.cu — batched Hamming search on the tensor cores: the list-major tile scan of Binary Flat / Binary IVF-Flat.
//
// ham(q, x) = popc(q) + popc(x) - 2 popc(q AND x).  The pair term is one BMMA per 16 rows x 8 queries x 256 bits
// (mma.sync m16n8k256 .and.popc, exact int32); popc(x) is summed from the A fragments while a row tile is in flight and
// popc(q) once per query.  Distances are exact integers, so unlike the float tile scan nothing is certified or re-scored:
//   bt_prep_queries_kernel  pad queries from w to w8 = round_up(w, 8) words, popc(q)
//   (tc_plan_pairs)         probes -> (list, query) pairs -> work items, shared with the float tile scan
//   bt_scan_kernel          persistent tile kernel: mode 0 writes the distances of each sampled span's first TC_SAMPLE rows,
//                           mode 1 captures every eligible row with dist <= tau_q
//   bt_tau_kernel           tau_q = k-th smallest sampled distance over eligible sampled rows (+inf when fewer than k)
//   bt_final_kernel         per query: top-k by (distance, id) over the captured rows (BlockSelect)
// A query whose capture overflowed or whose tau is +inf is re-run on the exact scan.  See DESIGN.md 4.8.
#include <algorithm>
#include <climits>
#include <mutex>

#include "binary_tile.cuh"
#include "scan_kernels.cuh"
#include "warp_select.cuh"

namespace b200vs {

namespace {

constexpr int BT_THREADS = 256;  // 8 warps: 4 row groups of 16 rows x 2 halves of the query block
constexpr int BT_BM = 64;        // rows per tile (accumulators per warp: 16 rows x N / 2 queries, at most 32 registers)
constexpr int BT_KW = 8;         // 32-bit words per K block (256 bits: one m16n8k256)
constexpr int BT_RS = 12;        // shared-memory row stride in words: 16-byte aligned, conflict-free fragment loads
constexpr int BT_STAGES = 4;     // cp.async ring depth (row tile + query block per stage)
constexpr int BT_A_WORDS = BT_BM * BT_RS, BT_B_WORDS = TC_NQT * BT_RS;
constexpr size_t BT_SMEM = (size_t)BT_STAGES * (BT_A_WORDS + BT_B_WORDS) * 4;
constexpr int BT_PL = 8192;  // sampled spans one query's threshold kernel stages
#define BT_INF __int_as_float(0x7f800000)

// one thread per (query, word of w8): zero padding past w; popc(q) accumulated per query
__global__ void bt_prep_queries_kernel(const uint32_t* __restrict__ q, long long nq, int w, int w8, uint32_t* __restrict__ q8, int* qpop) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq * w8) return;
  const long long r = i / w8;
  const int j = (int)(i % w8);
  const uint32_t v = j < w ? q[r * w + j] : 0u;
  q8[i] = v;
  if (v) atomicAdd(qpop + r, __popc(v));
}

__device__ __forceinline__ void cp_async16z(uint32_t* dst, const void* src, bool pred) {  // zero fill when !pred
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src), "r"(pred ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async4z(uint32_t* dst, const void* src, bool pred) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src), "r"(pred ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void bmma_and_popc(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

struct BtParams {
  const uint32_t* rows;  // arena words [arena rows, w]
  const long long* ids;
  const long long* list_off;
  int w, kblocks;              // stored words per row; 256-bit K blocks (w8 / 8)
  const uint32_t* qws;         // gathered queries [npairs + TC_NQT, w8]
  const int* qpop;             // [nq] popc(q)
  const TcItem* items;
  const int* totals;           // [0] n_items  [2] n_sample_items
  const int* sample_list;
  int* work_counter;
  const int* pair_query;
  float* sample;               // mode 0: [sample items, TC_NQT, TC_SAMPLE] distances, +inf for rows that are not eligible
  const float* tau;            // mode 1: [nq]
  unsigned long long* cand;    // mode 1: [nq, cap] (dist << 32 | arena row)
  int* cand_cnt;
  int cap;
  FilterDev filt;
};

// Stage step (tile t, K block kb) of an item into ring slot st: the row tile (A, zero past the item's rows and past w)
// and the item's query block (B, N rows of w8 words: always whole 16-byte chunks).
template <int N>
__device__ __forceinline__ void bt_stage(const BtParams& p, const TcItem& I, long long base_row, int rows, int t, int kb, uint32_t* sA, uint32_t* sB) {
  const int r0 = t * BT_BM;
  const int k0 = kb * BT_KW;
  if ((p.w & 3) == 0) {  // 16-byte aligned rows: two chunks per row, each either inside w or past it
    if (threadIdx.x < 2 * BT_BM) {
      const int r = threadIdx.x >> 1, c = threadIdx.x & 1;
      const bool ok = r0 + r < rows && k0 + 4 * c < p.w;
      const uint32_t* src = ok ? p.rows + (size_t)(base_row + r0 + r) * p.w + k0 + 4 * c : p.rows;
      cp_async16z(sA + r * BT_RS + 4 * c, src, ok);
    }
  } else {
#pragma unroll
    for (int i = 0; i < BT_BM * BT_KW / BT_THREADS; ++i) {
      const int e = threadIdx.x + i * BT_THREADS, r = e >> 3, j = e & 7;
      const bool ok = r0 + r < rows && k0 + j < p.w;
      const uint32_t* src = ok ? p.rows + (size_t)(base_row + r0 + r) * p.w + k0 + j : p.rows;
      cp_async4z(sA + r * BT_RS + j, src, ok);
    }
  }
  const int w8 = p.kblocks * BT_KW;
  for (int e = threadIdx.x; e < 2 * N; e += BT_THREADS) {
    const int n = e >> 1, c = e & 1;
    cp_async16z(sB + n * BT_RS + 4 * c, p.qws + (size_t)(I.pair_begin + n) * w8 + k0 + 4 * c, true);
  }
}

// One work item, N = query columns of the B block (16 / 32 / 64 / 128).  The (tile, K block) steps of the item run through
// one cp.async ring, so the next tile's loads overlap this tile's epilogue.  Warp w owns rows [16 (w % 4), 16 (w % 4) + 16)
// of each tile and query columns [NH (w / 4), NH (w / 4) + NH), NH = N / 2; its accumulators are rows g and g + 8
// (g = lane / 4) by columns 8j + 2 (lane % 4) + {0, 1} of that half.
template <int MODE, int N>
__device__ __forceinline__ void bt_item(const BtParams& p, const TcItem& I, uint32_t* ring, const int* s_q, const int* s_tau,
                                        const int* s_qpop, unsigned long long* hit_key, int* hit_q, int* hit_n) {
  constexpr int NH = N / 2, NT = NH / 8;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tig = lane & 3;
  const int rg = warp & 3, n0 = (warp >> 2) * NH;
  const long long base_row = p.list_off[I.list] + I.row_begin;
  int rows = I.row_end - I.row_begin;
  if (MODE == 0) rows = min(rows, TC_SAMPLE);
  const int ntiles = (rows + BT_BM - 1) / BT_BM;
  const int nsteps = ntiles * p.kblocks;
  auto sA = [&](int st) { return ring + st * (BT_A_WORDS + BT_B_WORDS); };
  auto sB = [&](int st) { return ring + st * (BT_A_WORDS + BT_B_WORDS) + BT_A_WORDS; };
#pragma unroll
  for (int s = 0; s < BT_STAGES - 1; ++s) {
    if (s < nsteps) bt_stage<N>(p, I, base_row, rows, s / p.kblocks, s % p.kblocks, sA(s), sB(s));
    cp_async_commit();
  }
  int acc[NT][4];
  int pop0 = 0, pop1 = 0;  // popc of rows g and g + 8 (this lane's words)
  for (int s = 0; s < nsteps; ++s) {
    const int t = s / p.kblocks, kb = s % p.kblocks;
    cp_async_wait<BT_STAGES - 2>();
    __syncthreads();  // step s has landed for every thread, and every warp is done with the slot refilled below
    {
      const int f = s + BT_STAGES - 1;
      if (f < nsteps) bt_stage<N>(p, I, base_row, rows, f / p.kblocks, f % p.kblocks, sA(f % BT_STAGES), sB(f % BT_STAGES));
      cp_async_commit();
    }
    if (kb == 0) {
#pragma unroll
      for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0;
      pop0 = pop1 = 0;
    }
    const int r = t * BT_BM + rg * 16;  // first row of this warp within the item
    if (r < rows) {
      const uint32_t* a = sA(s % BT_STAGES) + (rg * 16 + g) * BT_RS;
      const uint32_t* b = sB(s % BT_STAGES) + (n0 + g) * BT_RS;
      const uint32_t a0 = a[tig], a1 = a[8 * BT_RS + tig], a2 = a[4 + tig], a3 = a[8 * BT_RS + 4 + tig];
      pop0 += __popc(a0) + __popc(a2);
      pop1 += __popc(a1) + __popc(a3);
#pragma unroll
      for (int j = 0; j < NT; ++j) bmma_and_popc(acc[j], a0, a1, a2, a3, b[8 * j * BT_RS + tig], b[8 * j * BT_RS + 4 + tig]);
    }
    if (kb != p.kblocks - 1) continue;
    // epilogue of tile t (sample rows past the item are written as +inf, so warps without rows still run it in mode 0)
    if (MODE == 1 && r >= rows) continue;
    if (MODE == 0 && rg * 16 >= TC_SAMPLE) continue;
    pop0 += __shfl_xor_sync(0xffffffffu, pop0, 1); pop0 += __shfl_xor_sync(0xffffffffu, pop0, 2);
    pop1 += __shfl_xor_sync(0xffffffffu, pop1, 1); pop1 += __shfl_xor_sync(0xffffffffu, pop1, 2);
    // distances in place: acc[j][2h + c] = ham(row g + 8h, column n0 + 8j + 2 tig + c)
    const int lim = I.nq - n0 - 2 * tig;  // columns 8j + c < lim are queries of the item
    bool valid[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int rr = r + g + 8 * h;
      valid[h] = rr < rows;
      if (valid[h]) { const long long id = p.ids[base_row + rr]; valid[h] = id >= 0 && filter_pass(p.filt, id); }
    }
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int pq = 8 * j + c < lim ? s_qpop[n0 + 2 * tig + 8 * j + c] : 0;
        acc[j][c] = pop0 + pq - 2 * acc[j][c];
        acc[j][2 + c] = pop1 + pq - 2 * acc[j][2 + c];
      }
    if constexpr (MODE == 0) {
      float* sp = p.sample + ((size_t)I.sample_slot * TC_NQT + n0 + 2 * tig) * TC_SAMPLE + r + g;
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c)
          if (8 * j + c < lim)
#pragma unroll
            for (int h = 0; h < 2; ++h) sp[(8 * j + c) * TC_SAMPLE + 8 * h] = valid[h] ? (float)acc[j][2 * h + c] : BT_INF;
    } else {
      // hits are rare: a bit mask first, then one pass per hit
      uint32_t hits = 0;
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          // columns past the item's queries hold garbage, negative values included (> -2^17): never hits
          const int tq = 8 * j + c < lim ? s_tau[n0 + 2 * tig + 8 * j + c] : INT_MIN;
#pragma unroll
          for (int h = 0; h < 2; ++h)
            if (valid[h] && acc[j][2 * h + c] <= tq) hits |= 1u << (4 * j + 2 * h + c);
        }
      while (hits) {
        const int b = __ffs(hits) - 1;
        hits &= hits - 1;
        int dist = 0;
#pragma unroll
        for (int i = 0; i < 4 * NT; ++i) if (i == b) dist = acc[i >> 2][i & 3];
        const int h = (b >> 1) & 1, n = n0 + 2 * tig + 8 * (b >> 2) + (b & 1);
        const int q = s_q[n];
        const unsigned long long key = ((unsigned long long)(uint32_t)dist << 32) | (unsigned long long)(uint32_t)(base_row + r + g + 8 * h);
        const int hh = atomicAdd(hit_n, 1);
        if (hh < TC_HITS) { hit_key[hh] = key; hit_q[hh] = q; }
        else {  // staging full: write through
          const int sl = atomicAdd(p.cand_cnt + q, 1);
          if (sl < p.cap) p.cand[(size_t)q * p.cap + sl] = key;
        }
      }
    }
  }
  cp_async_wait<0>();
}

// Persistent: each CTA claims work items with one atomicAdd until the counter passes the item count.
template <int MODE>
__global__ void __launch_bounds__(BT_THREADS, 2) bt_scan_kernel(const BtParams p) {
  extern __shared__ __align__(16) uint32_t ring[];
  __shared__ int s_q[TC_NQT], s_qpop[TC_NQT];
  __shared__ int s_tau[TC_NQT];  // capture: tau_q (an integer), -1 when tau_q = +inf
  __shared__ int s_item;
  // capture staging, one buffer per warp, flushed when the item ends (as in the float tile kernel)
  __shared__ unsigned long long s_hit_key[BT_THREADS / 32][TC_HITS];
  __shared__ int s_hit_q[BT_THREADS / 32][TC_HITS];
  __shared__ int s_hit_n[BT_THREADS / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nwork = MODE == 0 ? p.totals[2] : p.totals[0];
  if (threadIdx.x < BT_THREADS / 32) s_hit_n[threadIdx.x] = 0;
  for (;;) {
    __syncthreads();  // the previous item is finished by every warp
    if (threadIdx.x == 0) {
      const int w = atomicAdd(p.work_counter, 1);
      s_item = w < nwork ? (MODE == 0 ? p.sample_list[w] : w) : -1;
    }
    __syncthreads();
    const int it = s_item;
    if (it < 0) break;
    const TcItem I = p.items[it];
    if (threadIdx.x < I.nq) {
      const int q = p.pair_query[I.pair_begin + threadIdx.x];
      s_q[threadIdx.x] = q;
      s_qpop[threadIdx.x] = p.qpop[q];
      const float tq = MODE == 1 ? p.tau[q] : 0.f;
      s_tau[threadIdx.x] = tq < BT_INF ? (int)tq : -1;  // an unthresholded query captures nothing: the exact scan answers it
    }
    // (the first barrier of the item's step loop publishes s_q / s_qpop / s_tau)
    if (I.nq <= 16) bt_item<MODE, 16>(p, I, ring, s_q, s_tau, s_qpop, s_hit_key[warp], s_hit_q[warp], &s_hit_n[warp]);
    else if (I.nq <= 32) bt_item<MODE, 32>(p, I, ring, s_q, s_tau, s_qpop, s_hit_key[warp], s_hit_q[warp], &s_hit_n[warp]);
    else if (I.nq <= 64) bt_item<MODE, 64>(p, I, ring, s_q, s_tau, s_qpop, s_hit_key[warp], s_hit_q[warp], &s_hit_n[warp]);
    else bt_item<MODE, 128>(p, I, ring, s_q, s_tau, s_qpop, s_hit_key[warp], s_hit_q[warp], &s_hit_n[warp]);
    if (MODE == 1) {  // flush this warp's staged hits
      __syncwarp();
      const int nh = min(s_hit_n[warp], TC_HITS);
      for (int i = lane; i < nh; i += 32) {
        const int q = s_hit_q[warp][i];
        const int sl = atomicAdd(p.cand_cnt + q, 1);
        if (sl < p.cap) p.cand[(size_t)q * p.cap + sl] = s_hit_key[warp][i];
      }
      __syncwarp();
      if (lane == 0) s_hit_n[warp] = 0;
      __syncwarp();
    }
  }
}

// One CTA per query: tau_q = the k-th smallest finite sampled distance of the query's probed lists, +inf when fewer than k
// (or more sampled spans than BT_PL, which the dispatch rules out).  Sampled rows that are tombstoned or filtered out hold
// +inf, so they never lower tau below the k-th distance of the eligible rows, and every row of the exact top-k has
// dist <= tau.  A query with tau = +inf is not captured (the exact scan answers it).
__global__ void __launch_bounds__(SCAN_THREADS)
bt_tau_kernel(const long long* __restrict__ probes, const int* __restrict__ pos, const int* __restrict__ cnt, const int* __restrict__ item_off,
              const int* __restrict__ list_len, const TcItem* __restrict__ items, int nprobe, const float* __restrict__ sample, int k, float* tau) {
  __shared__ int s_pairs[BT_PL];
  __shared__ BlockSelShared S;
  __shared__ int s_np, s_fin;
  const int q = blockIdx.x;
  if (threadIdx.x == 0) { s_np = 0; s_fin = 0; }
  __syncthreads();
  for (int j = threadIdx.x; j < nprobe; j += blockDim.x) {
    const long long l = probes[(size_t)q * nprobe + j];
    if (l < 0) continue;
    const int len = list_len[l];
    if (len <= 0) continue;
    const int ng = (cnt[l] + TC_NQT - 1) / TC_NQT;
    const int ps = pos[(size_t)q * nprobe + j];
    const int g = ps / TC_NQT, n = ps % TC_NQT;
    const int nspan = (len + TC_SPAN - 1) / TC_SPAN;
    const int base = atomicAdd(&s_np, nspan);
    for (int sp = 0; sp < nspan && base + sp < BT_PL; ++sp)
      s_pairs[base + sp] = items[item_off[l] + sp * (TC_SPAN / TC_CHUNK) * ng + g].sample_slot * TC_NQT + n;
  }
  __syncthreads();
  const int np = s_np;
  if (np > BT_PL) { if (threadIdx.x == 0) tau[q] = BT_INF; return; }
  const int tot = np * TC_SAMPLE;
  auto sampled = [&](int i) { return sample[(size_t)s_pairs[i / TC_SAMPLE] * TC_SAMPLE + i % TC_SAMPLE]; };
  int c = 0;
  for (int i = threadIdx.x; i < tot; i += blockDim.x) c += sampled(i) < BT_INF ? 1 : 0;
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_fin, c);
  __syncthreads();
  if (s_fin < k) { if (threadIdx.x == 0) tau[q] = BT_INF; return; }
  const uint32_t kth = block_kth_key_any(k, S, [&](auto f) {
    for (int i = threadIdx.x; i < tot; i += blockDim.x) { const float v = sampled(i); if (v < BT_INF) f(f2ord(v)); }
  });
  if (threadIdx.x == 0) tau[q] = ord2f(kth);
}

// One CTA per query: the exact top-k by (distance, id) of the captured rows.  flags[q] = 1 (exact re-run) when the capture
// overflowed or tau is +inf; the re-run writes that query's whole output row.
__global__ void __launch_bounds__(SCAN_THREADS)
bt_final_kernel(const unsigned long long* __restrict__ cand, const int* __restrict__ cand_cnt, int cap, const float* __restrict__ tau,
                const long long* __restrict__ ids, int k, int pool_cap, float* out_dist, long long* out_ids, int* flags) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int q = blockIdx.x;
  const int total = cand_cnt[q];
  if (total > cap || !(tau[q] < BT_INF)) { if (threadIdx.x == 0) flags[q] = 1; return; }
  const unsigned long long* c = cand + (size_t)q * cap;
  BlockSelect sel;
  sel.init(smem, pool_cap, k);
  for (int base = 0; base < total; base += blockDim.x) {
    sel.maybe_prune(blockDim.x);
    const int i = base + threadIdx.x;
    if (i < total) {
      const unsigned long long e = c[i];
      const uint32_t key = f2ord((float)(uint32_t)(e >> 32));
      const long long id = ids[(uint32_t)e];
      if (sel.passes(key, id)) sel.push(key, id);
    }
  }
  sel.prune();
  const int have = *sel.count;
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    out_dist[(size_t)q * k + i] = i < have ? ord2f(sel.kd[i]) : 0.f;
    out_ids[(size_t)q * k + i] = i < have ? sel.kid[i] : -1;
  }
  if (threadIdx.x == 0) flags[q] = 0;
}

std::mutex g_bt_mu;
int g_bt_slots[64] = {0};  // persistent CTAs per device (SMs x resident CTAs per SM)

int bt_slots(int device) {
  if (device < 0 || device >= 64) fail(B200VS_EILLEGAL_PARAMETERS, "bad CUDA device ordinal");
  std::lock_guard<std::mutex> g(g_bt_mu);
  if (!g_bt_slots[device]) {
    int n = 0;
    B200VS_CUDA(cudaSetDevice(device));
    B200VS_CUDA(cudaFuncSetAttribute(bt_scan_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BT_SMEM));
    B200VS_CUDA(cudaFuncSetAttribute(bt_scan_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BT_SMEM));
    B200VS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, bt_scan_kernel<1>, BT_THREADS, BT_SMEM));
    g_bt_slots[device] = device_sm_count(device) * std::max(1, n);
  }
  return g_bt_slots[device];
}

}  // namespace

bool bt_eligible(const TcView& v, int64_t nq, int k, int nprobe, double cand, const SearchCtx& sc) {
  if (sc.exact_only || nq < 16 || k > 128) return false;
  // The tile scan costs ~0.1 ms of planning, sampling and selection before it saves anything, and a threshold needs
  // k eligible rows among the 1 / 64 it samples.  Measured on the H100 (DESIGN.md 4.8), it beats the exact scan once
  // nq x candidate rows per query >= 2^23 (x k / 32 for k > 32: capture and final select grow with k) and the
  // candidates are at least 256 k rows; below that the exact scan is faster.
  if (cand < 256.0 * k) return false;
  if ((double)nq * cand < 8388608.0 * std::max(1.0, k / 32.0)) return false;
  // sampled spans of one query fit the threshold kernel's staging
  if ((int64_t)nprobe * ((v.max_chunks_per_list + TC_SPAN / TC_CHUNK - 1) / (TC_SPAN / TC_CHUNK)) > BT_PL) return false;
  return tc_plan_fits(v, nq, nprobe);
}

void bt_search(IndexBase* ix, const TcView& v, int w, int64_t nq, const uint32_t* q, int k, const long long* probes, int nprobe,
               const ScanJob& exact, float* out_dist, long long* out_ids, cudaStream_t s) {
  auto& S = ix->scratch;
  const SearchCtx& sc = *exact.sc;
  const int w8 = (w + BT_KW - 1) / BT_KW * BT_KW;
  const int cap = tc_cand_cap(k);
  ix->phase(IndexBase::PH_PLAN, s);
  uint32_t* q8 = S.alloc<uint32_t>((size_t)nq * w8);
  int* qpop = S.alloc<int>(nq);
  B200VS_CUDA(cudaMemsetAsync(qpop, 0, (size_t)nq * 4, s));
  bt_prep_queries_kernel<<<(unsigned)cdiv(nq * w8, 256), 256, 0, s>>>(q, nq, w, w8, q8, qpop);
  ix->launch_count(1);
  const TcPairs P = tc_plan_pairs(ix, v, nq, probes, nprobe, q8, w8 * 4, s);
  float* sample = S.alloc<float>((size_t)P.sbound * TC_NQT * TC_SAMPLE);
  float* tau = S.alloc<float>(nq);
  unsigned long long* cand = S.alloc<unsigned long long>((size_t)nq * cap);
  int* cand_cnt = S.alloc<int>(nq);
  int* flags = S.alloc<int>(nq);
  int* qmap = S.alloc<int>(nq);
  int* qcount = S.alloc<int>(1);
  B200VS_CUDA(cudaMemsetAsync(cand_cnt, 0, (size_t)nq * 4, s));

  BtParams p{};
  p.rows = reinterpret_cast<const uint32_t*>(v.vecs); p.ids = v.ids; p.list_off = v.list_off; p.w = w; p.kblocks = w8 / BT_KW;
  p.qws = static_cast<const uint32_t*>(P.bws); p.qpop = qpop;
  p.items = P.items; p.totals = P.totals; p.sample_list = P.sample_list; p.pair_query = P.pair_query;
  p.sample = sample; p.tau = tau; p.cand = cand; p.cand_cnt = cand_cnt; p.cap = cap;
  p.filt.has_range = sc.has_range; p.filt.negate = sc.negate; p.filt.rmin = sc.rmin; p.filt.rmax = sc.rmax;
  p.filt.sorted_ids = sc.sorted_ids_dev; p.filt.n_ids = sc.n_ids;
  const int slots = bt_slots(ix->device);
  auto grid = [&](int64_t bound) { return (unsigned)std::min<int64_t>(slots, std::max<int64_t>(1, bound)); };
  // 1) sample pass -> per-query thresholds
  p.work_counter = P.work;
  ix->phase(IndexBase::PH_SAMPLE, s);
  bt_scan_kernel<0><<<grid(P.sbound), BT_THREADS, BT_SMEM, s>>>(p);
  ix->phase(IndexBase::PH_TAU, s);
  bt_tau_kernel<<<(unsigned)nq, SCAN_THREADS, 0, s>>>(probes, P.pos, P.cnt, P.item_off, v.list_len, P.items, nprobe, sample, k, tau);
  // 2) capture pass: every probed list chunk streamed once per query group
  p.work_counter = P.work + 1;
  ix->phase(IndexBase::PH_CAPTURE, s);
  {
    ScopedKernelTimer timer(ix, s, ix->profiling);
    bt_scan_kernel<1><<<grid(P.bound), BT_THREADS, BT_SMEM, s>>>(p);
    timer.stop();
  }
  // 3) top-k of the captured rows
  ix->phase(IndexBase::PH_FINAL, s);
  const int pool = select_pool_cap(k, SCAN_THREADS);
  bt_final_kernel<<<(unsigned)nq, SCAN_THREADS, BlockSelect::smem_bytes(pool), s>>>(cand, cand_cnt, cap, tau, v.ids, k, pool, out_dist, out_ids, flags);
  tc_compact_flags(flags, (int)nq, qmap, qcount, s);
  B200VS_CUDA(cudaGetLastError());
  ix->launch_count(5);
  ix->stats[1] = nq;
  // 4) overflowed / unthresholded queries on the exact scan (device-side count: blocks beyond it exit at once)
  ix->phase(IndexBase::PH_FALLBACK, s);
  run_scan_mapped(ix, exact, nq, qmap, qcount, reinterpret_cast<const float*>(q), k, out_dist, nullptr, out_ids, nullptr, s);
  ix->phase(IndexBase::PH_OTHER, s);
  if (ix->profiling) {
    int h = 0, t[4] = {0, 0, 0, 0};
    B200VS_CUDA(cudaMemcpyAsync(&h, qcount, 4, cudaMemcpyDeviceToHost, s));
    B200VS_CUDA(cudaMemcpyAsync(t, P.totals, 16, cudaMemcpyDeviceToHost, s));
    B200VS_CUDA(cudaStreamSynchronize(s));
    ix->stats[2] = h;
    ix->stats[6] = t[0];  // work items of the capture pass
    ix->stats[7] = t[3];  // sum over items of (128-row tiles x padded query columns)
  }
}

}  // namespace b200vs
