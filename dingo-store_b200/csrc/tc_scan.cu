// tc_scan.cu — tensor-core candidate pass (see tc_scan.cuh for the contract, DESIGN.md for the proof sketch).
//
// Kernels:
//   tc_prep_queries_kernel   round queries to TF32 (RN), ||q||^2
//                            (tc_prep_queries_half_kernel: power-of-two scale + FP16 (RN), for the FP16 mirror)
//   tc_half_rows_kernel      the FP16 mirror of arena rows (power-of-two scale per row + FP16 RN)
//   tc_count_pairs_kernel    invert the probe table: how many queries probe each list
//   tc_plan_kernel           exclusive scans -> pair offsets, work-item offsets
//   tc_fill_pairs_kernel     gather the (rounded) queries of every list into one contiguous block
//   tc_items_kernel          emit work items (list chunk x query group) + the list of sampled items
//   tc_scan_kernel           *** the hot kernel: TMA -> smem ring -> wgmma (TF32 or FP16, register accumulators) -> epilogue ***
//   tc_range_tau_kernel      range mode: per-query capture threshold from the radius, widened by tc_eps
//   tc_tau_warp_kernel       per-query capture threshold from the sampled rows (warp radix select)
//                            (tc_tau_kernel: the block form for queries with more sampled spans than a warp stages)
//   tc_final_hybrid_kernel   per-query window select + exact FP32 (AVX-512 order) rerank + certification
//                            (tc_final_kernel: the streaming form for windows or query rows that do not fit; both
//                            have a range form that re-scores every captured row and keeps the hits)
//   tc_coarse_select_hybrid_kernel / tc_coarse_select_kernel
//                            coarse-quantiser finish: register-resident radix select + exact rerank of the window
//                            (tc_coarse_final_kernel: the streaming form for what they cannot finish)
//   tc_compact_flags_kernel  list of uncertified queries for the exact re-run
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <mutex>
#include <type_traits>

#include "scan_kernels.cuh"
#include "sm90_ptx.cuh"
#include "tc_scan.cuh"
#include "warp_select.cuh"

namespace b200vs {

using namespace ptx;

#define TC_INF __int_as_float(0x7f800000)

// ---------------------------------------------------------------------------------------------
// small helper kernels
// ---------------------------------------------------------------------------------------------
static __global__ void tc_prep_queries_kernel(const float* __restrict__ q, long long nq, int d, float* __restrict__ q32,
                                              float* __restrict__ qnorm) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= nq) return;
  const float* src = q + (size_t)w * d;
  float* dst = q32 + (size_t)w * d;
  float acc = 0.f;
  for (int i = lane; i < d; i += 32) {
    const float v = src[i];
    acc = fmaf(v, v, acc);
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    dst[i] = __uint_as_float(r);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) qnorm[w] = acc;
}

// error-compensated operands: hi = TF32 (low 13 mantissa bits cleared / rounded), lo = remainder
static __global__ void tc_prep_queries_split_kernel(const float* __restrict__ q, long long nq, int d, float* __restrict__ qhi,
                                                    float* __restrict__ qlo, float* __restrict__ qnorm) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= nq) return;
  float acc = 0.f;
  for (int i = lane; i < d; i += 32) {
    const float v = q[(size_t)w * d + i];
    acc = fmaf(v, v, acc);
    uint32_t r, r2;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    const float hi = __uint_as_float(r);
    const float lo = __fsub_rn(v, hi);  // exact
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r2) : "f"(lo));
    qhi[(size_t)w * d + i] = hi;
    qlo[(size_t)w * d + i] = __uint_as_float(r2);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) qnorm[w] = acc;
}
// FP16 operands: x * 2^-e rounded to nearest, with e chosen so that max |x_i| * 2^-e lies in [2^14, 2^15) (no overflow;
// underflow costs at most 2^-25 * 2^e <= 2^-39 max |x_i| per element).  Scaling by a power of two is exact in FP32, so
// the only rounding is the one to FP16 (DESIGN.md 4.2).  A zero vector keeps e = 0.
__device__ __forceinline__ int tc_half_exp(float maxabs) { return maxabs > 0.f ? ilogbf(maxabs) - 14 : 0; }

// one warp per row: dst = the scaled FP16 row, *scale = 2^e; returns <x, x> (FP32, this warp's order) to lane 0.
__device__ __forceinline__ float tc_half_row(const float* __restrict__ src, int d, __half* __restrict__ dst, float* scale) {
  const int lane = threadIdx.x & 31;
  float m = 0.f, acc = 0.f;
  for (int i = lane; i < d; i += 32) { const float v = src[i]; m = fmaxf(m, fabsf(v)); acc = fmaf(v, v, acc); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o)); acc += __shfl_xor_sync(0xffffffffu, acc, o); }
  const int e = tc_half_exp(m);
  for (int i = lane; i < d; i += 32) dst[i] = __float2half_rn(ldexpf(src[i], -e));
  if (lane == 0) *scale = ldexpf(1.f, e);
  return acc;
}

static __global__ void tc_prep_queries_half_kernel(const float* __restrict__ q, long long nq, int d, __half* __restrict__ qh,
                                                   float* __restrict__ qscale, float* __restrict__ qnorm) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= nq) return;
  const float n2 = tc_half_row(q + (size_t)w * d, d, qh + (size_t)w * d, qscale + w);
  if ((threadIdx.x & 31) == 0) qnorm[w] = n2;
}

static __global__ void tc_half_rows_kernel(const float* __restrict__ x, const long long* __restrict__ rows, long long n, int d,
                                           __half* __restrict__ half, float* __restrict__ scale) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= n) return;
  const long long r = rows ? rows[w] : w;
  tc_half_row(x + (size_t)r * d, d, half + (size_t)r * d, scale + r);
}
void launch_half_rows(const float* x, const long long* rows, int64_t n, int d, __half* half, float* scale, cudaStream_t s) {
  if (n <= 0) return;
  tc_half_rows_kernel<<<(unsigned)cdiv(n * 32, 256), 256, 0, s>>>(x, rows, n, d, half, scale);
  B200VS_CUDA(cudaGetLastError());
}

static __global__ void tc_split_rows_kernel(const float* __restrict__ x, long long n, float* __restrict__ hi, float* __restrict__ lo) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = x[i];
  const float h = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
  hi[i] = h;
  lo[i] = __fsub_rn(v, h);  // exact; the tensor core truncates it to TF32 (error <= 2^-20 |x|)
}
void launch_split_rows(const float* x, int64_t n, int d, float* hi, float* lo, cudaStream_t s) {
  const long long tot = (long long)n * d;
  if (tot <= 0) return;
  tc_split_rows_kernel<<<(unsigned)cdiv(tot, 256), 256, 0, s>>>(x, tot, hi, lo);
  B200VS_CUDA(cudaGetLastError());
}
// coarse pass: items = (row chunk) x (group of nqt <= TC_NQT queries); B rows are the query rows themselves
static __global__ void tc_coarse_items_kernel(int nrows, int nq, int chunk, int nqt, TcItem* items, int* totals) {
  const int nc = (nrows + chunk - 1) / chunk, ng = (nq + nqt - 1) / nqt;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) { totals[0] = nc * ng; totals[1] = nq; totals[2] = 0; }
  if (i >= nc * ng) return;
  const int ch = i / ng, g = i % ng;
  TcItem it;
  it.list = 0; it.row_begin = ch * chunk; it.row_end = min(nrows, (ch + 1) * chunk);
  it.pair_begin = g * nqt; it.nq = min(nqt, nq - g * nqt); it.sample_slot = -1; it.pad[0] = it.pad[1] = 0;
  items[i] = it;
}

static __global__ void tc_count_pairs_kernel(const long long* __restrict__ probes, long long n, int* cnt, int* pos) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long l = probes[i];
  pos[i] = l >= 0 ? atomicAdd(cnt + l, 1) : -1;
}

// A work item's nq queries fill a B tile of 16 << tc_bcols_log(nq) = 16 / 32 / 64 / 128 rows (the wgmma N), read through TcMaps::b[]
__device__ __forceinline__ int tc_bcols_log(int nq) { return nq <= 16 ? 0 : (nq <= 32 ? 1 : (nq <= 64 ? 2 : 3)); }

__device__ __forceinline__ int tc_items_of(int c, int len) {
  return (c > 0 && len > 0) ? ((c + TC_NQT - 1) / TC_NQT) * ((len + TC_CHUNK - 1) / TC_CHUNK) : 0;
}

// single block: exclusive scans over the lists
static __global__ void tc_plan_kernel(const int* __restrict__ cnt, const int* __restrict__ list_len, int nlist, int* pair_off,
                                      int* item_off, int* totals /*[0]=n_items [1]=n_pairs [2]=n_sample (zeroed here)*/) {
  __shared__ int s_pairs[1024], s_items[1024];
  const int t = threadIdx.x, T = blockDim.x;
  const int per = (nlist + T - 1) / T;
  const int b = t * per, e = min(nlist, b + per);
  int sp = 0, si = 0;
  for (int l = b; l < e; ++l) { sp += cnt[l]; si += tc_items_of(cnt[l], list_len[l]); }
  // block-wide exclusive scan of (sp, si): warp shuffles + one scan of the 32 warp totals
  const int lane = t & 31, wid = t >> 5;
  int ip = sp, ii = si;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int vp = __shfl_up_sync(0xffffffffu, ip, o), vi = __shfl_up_sync(0xffffffffu, ii, o);
    if (lane >= o) { ip += vp; ii += vi; }
  }
  if (lane == 31) { s_pairs[wid] = ip; s_items[wid] = ii; }
  __syncthreads();
  if (wid == 0) {
    int wp = lane < (T >> 5) ? s_pairs[lane] : 0, wi = lane < (T >> 5) ? s_items[lane] : 0;
    const int tp = wp, ti = wi;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int vp = __shfl_up_sync(0xffffffffu, wp, o), vi = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) { wp += vp; wi += vi; }
    }
    if (lane == 31) { totals[0] = wi; totals[1] = wp; totals[2] = 0; totals[3] = 0; }
    s_pairs[lane] = wp - tp; s_items[lane] = wi - ti;  // exclusive warp offsets
  }
  __syncthreads();
  sp = s_pairs[wid] + ip - sp; si = s_items[wid] + ii - si;  // exclusive prefix of this thread
  for (int l = b; l < e; ++l) {
    pair_off[l] = sp; item_off[l] = si;
    sp += cnt[l]; si += tc_items_of(cnt[l], list_len[l]);
  }
}

// one warp per (query, probe): place the pair and copy the rounded query row (row_bytes = d * 4 or d * 2, a multiple of 16)
static __global__ void tc_fill_pairs_kernel(const long long* __restrict__ probes, const int* __restrict__ pos,
                                            const int* __restrict__ pair_off, const int* __restrict__ list_len, long long n,
                                            int nprobe, int row_bytes, const void* __restrict__ qop, int* pair_query, void* bws) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const long long l = probes[w];
  if (l < 0 || list_len[l] <= 0) return;  // empty list (e.g. owned by another shard): no work item will read this row
  const int p = pair_off[l] + pos[w];
  const int q = (int)(w / nprobe);
  if (lane == 0) pair_query[p] = q;
  const uint4* src = reinterpret_cast<const uint4*>(static_cast<const char*>(qop) + (size_t)q * row_bytes);
  uint4* dst = reinterpret_cast<uint4*>(static_cast<char*>(bws) + (size_t)p * row_bytes);
  for (int i = lane; i < (row_bytes >> 4); i += 32) dst[i] = src[i];
}

// items of list l live at item_off[l] + chunk * ngroups + group  (the groups of one chunk are adjacent: the
// second group re-reads the chunk from L2 while it is hot)
static __global__ void tc_items_kernel(const int* __restrict__ cnt, const int* __restrict__ list_len,
                                       const int* __restrict__ pair_off, const int* __restrict__ item_off, int nlist, TcItem* items,
                                       int* totals, int* sample_list) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= nlist) return;
  const int c = cnt[l], len = list_len[l];
  if (c <= 0 || len <= 0) return;
  const int ng = (c + TC_NQT - 1) / TC_NQT, nc = (len + TC_CHUNK - 1) / TC_CHUNK;
  const int base = item_off[l];
  for (int ch = 0; ch < nc; ++ch)
    for (int g = 0; g < ng; ++g) {
      TcItem it;
      it.list = l;
      it.row_begin = ch * TC_CHUNK;
      it.row_end = min(len, (ch + 1) * TC_CHUNK);
      it.pair_begin = pair_off[l] + g * TC_NQT;
      it.nq = min(TC_NQT, c - g * TC_NQT);
      it.sample_slot = -1;
      if ((it.row_begin % TC_SPAN) == 0) {
        it.sample_slot = atomicAdd(totals + 2, 1);
        sample_list[it.sample_slot] = base + ch * ng + g;
      }
      it.pad[0] = it.pad[1] = 0;
      items[base + ch * ng + g] = it;
      // profiling aid: tensor-core work = 128-row tiles x padded query columns
      atomicAdd(totals + 3, ((it.row_end - it.row_begin + TC_BM - 1) / TC_BM) * (16 << tc_bcols_log(it.nq)));
    }
}

// ---------------------------------------------------------------------------------------------
// THE HOT KERNEL.  Persistent (one CTA per SM in its capture form), warp-specialised, dynamically scheduled:
//   warp 8 (one lane): scheduler + TMA producer — claims the next work item with one atomicAdd, publishes it through
//                      a 4-deep smem queue, then per K block loads the A tile = 128 list rows x 128 B (16 KB,
//                      EVICT_FIRST: streamed once) and the B tile = 16/32/64/128 gathered queries x 128 B (EVICT_LAST)
//   warps 0-7        : two consumer warpgroups; warpgroup g owns rows [64g, 64g + 64) of every 128-row tile.  Per K block
//                      4 x wgmma (M=64, N=16..128, K = 8 TF32 or 16 FP16) with the accumulators in registers, then the
//                      epilogue on those registers: undo the power-of-two scales (FP16), add ||x||^2, then sample / capture
//                      (staged in shared memory, flushed per item) / dense store.  The producer keeps filling the ring while
//                      the epilogue runs.
// HALF = false: K block = 32 floats of the FP32 rows; HALF = true: 64 halves of the FP16 mirror, so a row costs half the
// tile loads.  Algorithmic HBM bytes per item: rows x (d*4 + 4 + 8) (vector, norm, id), or rows x (d*2 + 4 + 4 + 8) on the
// mirror (+ scale), read exactly once.
//
// One form per mode and operand type (TcCfg<MODE>).  The capture form (mode 1) is the one above.  The sample pass (mode 0)
// only ever scores the first TC_SAMPLE rows of an item, so its form has one consumer warpgroup and a 3-stage ring of 32-row
// A boxes, without capture staging: three of its CTAs share an SM, so three times as many items' start-up round trips
// overlap.  The dense pass (mode 2: coarse quantiser, labelling, diagnostics) reads a small table from L2 item after item;
// its form has one consumer warpgroup on 64-row tiles, query groups of at most TC_DENSE_NQT and a 4-stage ring (two split
// K blocks), so three CTAs share an SM and the pass has three items per SM in flight instead of one.
// All forms run the same per-row wgmma sequence and epilogue (tc_mma_tile / tc_consume_item) on stages that start on a
// 1024-byte boundary, so a score does not depend on the form: a sampled score is bit for bit the score the capture pass
// computes for that (row, query).
// ---------------------------------------------------------------------------------------------
constexpr int TC_DENSE_NQT = 64;  // widest query group of the dense form (its B stage)

template <int Mode>
struct TcCfg {
  static constexpr int MODE = Mode;                 // 0 = sample, 1 = capture, 2 = dense (TcParams::mode)
  static constexpr int CWARPS = MODE == 1 ? 8 : 4;  // consumer warps (one or two warpgroups); the producer is warp CWARPS
  static constexpr int BM = CWARPS / 4 * 64;        // rows per tile: 64 per consumer warpgroup
  static constexpr int THREADS = CWARPS * 32 + 32;
  static constexpr int MIN_CTAS = MODE == 1 ? 1 : 3;  // CTAs per SM the launch bounds reserve registers for
  // TMA -> MMA ring.  Capture: 6 x 32 KB (+ 24 KB of capture staging: ~220 KB; the bytes in flight bound the HBM rate,
  // DESIGN §4.2).  Sample: 3 x (4 KB A box + 16 KB B tile) = 61 KB with the alignment slack.  Dense: 4 x (8 KB A tile +
  // 8 KB B tile) = 65 KB.  Every stride is a multiple of 1024, the period of the 128-byte swizzle.
  static constexpr int STAGES = MODE == 1 ? 6 : (MODE == 0 ? 3 : 4);
  static constexpr uint32_t A_STAGE = MODE == 0 ? TC_SAMPLE * 128 : BM * 128;
  static constexpr uint32_t B_STAGE = MODE == 2 ? TC_DENSE_NQT * 128 : TC_B_BYTES;
  static constexpr size_t SMEM = (size_t)STAGES * (A_STAGE + B_STAGE) + 1024;
};

template <int STAGES>
struct TcRing {  // a consumer's position in the TMA ring
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void next() {
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
};

// One 128-row tile: this warpgroup's 64 x N scores into acc.  Every consumer warp waits for and releases every stage,
// also when its warpgroup has no rows in the tile (mma = false).  In the sample form a stage holds 32 A rows, so the
// M = 64 wgmma also reads the 32 rows after them (the next stage, or the first B tile): their scores land in accumulator
// rows 32-63, which the epilogue never stores (as with the stale rows of a partly loaded capture stage).
template <bool HALF, int N, class C>
__device__ __forceinline__ void tc_mma_tile(const TcParams& p, int kblocks, bool mma, uint8_t* sA, uint8_t* sB, uint64_t* full_bar,
                                            uint64_t* empty_bar, TcRing<C::STAGES>& ring, float (&acc)[N / 2]) {
  const int lane = threadIdx.x & 31;
  const uint32_t a_off = (uint32_t)(threadIdx.x >> 7) * 64u * 128u;  // warpgroup g: rows [64g, 64g + 64)
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < kblocks; ++kb) {
    const int s_hi = ring.stage;
    mbar_wait(&full_bar[s_hi], ring.phase);
    ring.next();
    int s_lo = 0;
    const bool split = !HALF && C::MODE == 2 && p.split;
    if (split) {  // error-compensated pass: the "lo" operands ride in the next ring stage
      s_lo = ring.stage;
      mbar_wait(&full_bar[s_lo], ring.phase);
      ring.next();
    }
    if (mma) {
      const uint64_t adesc = make_desc_k128(smem_u32(sA + (size_t)s_hi * C::A_STAGE + a_off));
      const uint64_t bdesc = make_desc_k128(smem_u32(sB + (size_t)s_hi * C::B_STAGE));
      wgmma_fence_operands(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TC_BK / 8; ++k) {  // one 32-byte K step each
        if constexpr (HALF) wgmma_f16<N>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (kb | k) != 0 ? 1u : 0u);
        else wgmma_tf32<N>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (kb | k) != 0 ? 1u : 0u);
      }
      if (split) {  // + lo*hi + hi*lo into the same accumulator
        const uint64_t adesc_lo = make_desc_k128(smem_u32(sA + (size_t)s_lo * C::A_STAGE + a_off));
        const uint64_t bdesc_lo = make_desc_k128(smem_u32(sB + (size_t)s_lo * C::B_STAGE));
#pragma unroll
        for (int k = 0; k < TC_BK / 8; ++k) {
          wgmma_tf32<N>(acc, adesc_lo + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), 1u);
          wgmma_tf32<N>(acc, adesc + (uint64_t)(2 * k), bdesc_lo + (uint64_t)(2 * k), 1u);
        }
      }
      wgmma_commit();
      wgmma_wait_all();  // the MMAs have read the stage(s)
      wgmma_fence_operands(acc);
    }
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(&empty_bar[s_hi]);
      if (split) mbar_arrive(&empty_bar[s_lo]);
    }
  }
}

// One work item on the consumer warps; N = query columns of the B tile (16 / 32 / 64 / 128).
// Thread layout of the accumulators: rows row0 and row0 + 8 of the tile, columns 8j + col0 + {0, 1}.
template <bool HALF, int N, class C>
__device__ __forceinline__ void tc_consume_item(const TcParams& p, const TcItem& I, int kblocks, uint8_t* sA, uint8_t* sB,
                                                uint64_t* full_bar, uint64_t* empty_bar, TcRing<C::STAGES>& ring, const float* s_tau,
                                                const int* s_q, const float* s_qs, unsigned long long* hit_key, int* hit_q, int* hit_n) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), col0 = 2 * (lane & 3);
  const long long list_base = p.list_off[I.list];
  int rows = I.row_end - I.row_begin;
  if constexpr (C::MODE == 0) rows = min(rows, TC_SAMPLE);
  const int ntiles = (rows + C::BM - 1) / C::BM;
  for (int t = 0; t < ntiles; ++t) {
    // row metadata first: its loads overlap the MMAs.  The id and norm loads do not depend on each other, and the masks
    // that read the id are applied after the MMAs, so no warp waits for a global round trip before its first wgmma
    bool inrange[2], valid[2];
    long long arow[2], id[2];
    float nrm[2], hs[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = t * C::BM + row0 + 8 * h;
      inrange[h] = r < rows;
      arow[h] = list_base + I.row_begin + r;
      id[h] = -1;
      nrm[h] = 0.f;
      hs[h] = 1.f;
      if (inrange[h]) {
        id[h] = p.ids[arow[h]];
        if (p.l2) nrm[h] = p.norms[arow[h]];
        if constexpr (HALF) hs[h] = p.hscale[arow[h]];
      }
    }
    float acc[N / 2];
    const bool mma = t * C::BM + wg * 64 < rows;  // else this warpgroup's half of the last tile holds no item rows
    tc_mma_tile<HALF, N, C>(p, kblocks, mma, sA, sB, full_bar, empty_bar, ring, acc);
    if (!mma) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      valid[h] = inrange[h] && id[h] >= 0 && filter_pass(p.filt, id[h]);
      if (!valid[h]) nrm[h] = 0.f;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = t * C::BM + row0 + 8 * h;  // row within the item
#pragma unroll
      for (int j = 0; j < N / 8; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int n = 8 * j + col0 + c;
          if (n < I.nq) {
            // FP16: both scales are powers of two, so hs * qs and the product with the accumulator are exact while they
            // stay normal; below that they underflow (to 0 under 2^-149), which tc_eps's absolute term covers
            const float dot = HALF ? acc[4 * j + 2 * h + c] * (hs[h] * s_qs[n]) : acc[4 * j + 2 * h + c];
            const float score = p.l2 ? fmaf(-2.f, dot, nrm[h]) : -dot;
            if constexpr (C::MODE == 0) {
              if (t == 0 && r < TC_SAMPLE) p.sample[((size_t)I.sample_slot * TC_NQT + n) * TC_SAMPLE + r] = valid[h] ? score : TC_INF;
            } else if constexpr (C::MODE == 1) {
              if (valid[h] && score <= s_tau[n]) {
                const int q = s_q[n];
                const unsigned long long key = ((unsigned long long)f2ord(score) << 32) | (unsigned long long)(uint32_t)arow[h];
                const int hh = atomicAdd(hit_n, 1);
                if (hh < TC_HITS) { hit_key[hh] = key; hit_q[hh] = q; }
                else {  // staging full: write through
                  const int sl = atomicAdd(p.cand_cnt + q, 1);
                  if (sl < p.cap) p.cand[(size_t)q * p.cap + sl] = key;
                }
              }
            } else if (inrange[h]) {
              p.dense[(size_t)s_q[n] * p.dense_ld + (I.row_begin + r)] = valid[h] ? score : TC_INF;
            }
          }
        }
    }
  }
}

// The tile kernel's TMA descriptors (make_tc_maps): a / a32 = the A rows in 128-row / 32-row boxes, b[i] = the B block in
// 16 << i row boxes, a_lo / b_lo = the split pass's lo operands (the hi maps again when there are none).  The kernel only
// takes the maps' addresses: a copy would land in local memory, where TMA cannot read it.
struct TcMaps {
  CUtensorMap a, a32, b[4], a_lo, b_lo[4];
};

// MODE = the pass this form runs (TcParams::mode: 0 sample, 1 capture, 2 dense).
template <bool HALF, int MODE>
__global__ void __launch_bounds__(TcCfg<MODE>::THREADS, TcCfg<MODE>::MIN_CTAS)
tc_scan_kernel(const __grid_constant__ TcMaps maps, const TcParams p) {
  using C = TcCfg<MODE>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = smem;
  uint8_t* sB = smem + (size_t)C::STAGES * C::A_STAGE;
  __shared__ __align__(8) uint64_t full_bar[C::STAGES], empty_bar[C::STAGES];
  __shared__ __align__(8) uint64_t sched_full[TC_SQ], sched_empty[TC_SQ];
  __shared__ int s_sched[TC_SQ];
  __shared__ float s_tau[2][TC_NQT];
  __shared__ int s_q[2][TC_NQT];
  __shared__ float s_qs[2][TC_NQT];
  // capture staging, one buffer per consumer warp: hits are appended with a shared-memory atomic and written out
  // (one global atomicAdd per hit, a whole warp of them in flight) when the item ends, so the score loop never
  // waits on a global round trip.  The other forms capture nothing and keep a one-entry placeholder.
  constexpr int HW = MODE == 1 ? C::CWARPS : 1, HN = MODE == 1 ? TC_HITS : 1;
  __shared__ unsigned long long s_hit_key[HW][HN];
  __shared__ int s_hit_q[HW][HN];
  __shared__ int s_hit_n[HW];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x < HW) s_hit_n[threadIdx.x] = 0;
  if (warp == C::CWARPS && lane == 0) {
    prefetch_tmap(&maps.a); prefetch_tmap(&maps.a32);
    for (int i = 0; i < 4; ++i) prefetch_tmap(&maps.b[i]);
    for (int i = 0; i < C::STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], C::CWARPS); }
    for (int i = 0; i < TC_SQ; ++i) { mbar_init(&sched_full[i], 1); mbar_init(&sched_empty[i], C::CWARPS); }
    fence_barrier_init();
  }
  __syncthreads();
  const int nwork = MODE == 0 ? p.totals[2] : p.totals[0];
  const int kbk = HALF ? 2 * TC_BK : TC_BK;  // elements per K block (128 B)
  const int kblocks = (p.d + kbk - 1) / kbk;

  if (warp == C::CWARPS) {
    if (lane == 0) {  // ---------------- scheduler + TMA producer ----------------
      int stage = 0, slot = 0;
      uint32_t phase = 0, sphase = 0;
      for (;;) {
        mbar_wait(&sched_empty[slot], sphase ^ 1);
        const int w = atomicAdd(p.work_counter, 1);
        const int it = w < nwork ? (MODE == 0 ? p.sample_list[w] : w) : -1;
        s_sched[slot] = it;
        mbar_arrive(&sched_full[slot]);
        if (++slot == TC_SQ) { slot = 0; sphase ^= 1; }
        if (it < 0) break;
        const TcItem I = p.items[it];
        const long long base_row = p.list_off[I.list] + I.row_begin;
        int rows = I.row_end - I.row_begin;
        if (MODE == 0) rows = min(rows, TC_SAMPLE);
        const int ntiles = (rows + C::BM - 1) / C::BM;
        const int bl = tc_bcols_log(I.nq);
        const CUtensorMap* tb = &maps.b[bl];
        const CUtensorMap* ta = MODE == 0 ? &maps.a32 : &maps.a;  // 32-row sample box, else the whole C::BM-row tile
        const uint32_t bytes = C::A_STAGE + (16u << bl) * 128u;
        const CUtensorMap* tbl = &maps.b_lo[bl];
        for (int t = 0; t < ntiles; ++t)
          for (int kb = 0; kb < kblocks; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            // last tile of a list: fetch only the 32-row boxes that hold list rows (the rest of the stage keeps stale
            // data, whose scores the epilogue masks) instead of streaming up to 127 rows of the neighbouring list
            const int trows = rows - t * C::BM;
            const int nbox = (MODE == 1 && trows <= C::BM - TC_SAMPLE) ? (trows + TC_SAMPLE - 1) / TC_SAMPLE : 0;
            const uint32_t saved = nbox ? TC_A_BYTES - (uint32_t)nbox * (TC_SAMPLE * 128) : 0u;
            mbar_arrive_expect_tx(&full_bar[stage], bytes - saved);
            if (nbox) {
              for (int j = 0; j < nbox; ++j)
                tma_load_2d(sA + (size_t)stage * C::A_STAGE + (size_t)j * (TC_SAMPLE * 128), &maps.a32, &full_bar[stage], kb * kbk,
                            (int)(base_row + (long long)t * TC_BM + j * TC_SAMPLE), kEvictFirst);
            } else
            tma_load_2d(sA + (size_t)stage * C::A_STAGE, ta, &full_bar[stage], kb * kbk, (int)(base_row + (long long)t * C::BM), kEvictFirst);
            tma_load_2d(sB + (size_t)stage * C::B_STAGE, tb, &full_bar[stage], kb * kbk, I.pair_begin, kEvictLast);
            if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
            if (!HALF && MODE == 2 && p.split) {  // error-compensated pass: the "lo" operands ride in the next ring stage
              mbar_wait(&empty_bar[stage], phase ^ 1);
              mbar_arrive_expect_tx(&full_bar[stage], bytes);
              tma_load_2d(sA + (size_t)stage * C::A_STAGE, &maps.a_lo, &full_bar[stage], kb * kbk, (int)(base_row + (long long)t * C::BM), kEvictFirst);
              tma_load_2d(sB + (size_t)stage * C::B_STAGE, tbl, &full_bar[stage], kb * kbk, I.pair_begin, kEvictLast);
              if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
            }
          }
      }
    }
    return;
  }
  // ---------------- consumers: warps 0 .. CWARPS - 1 ----------------
  TcRing<C::STAGES> ring;
  uint32_t sphase = 0;
  int slot = 0;
  for (int icount = 0;; ++icount) {
    mbar_wait(&sched_full[slot], sphase);
    const int it = s_sched[slot];
    __syncwarp();
    if (lane == 0) mbar_arrive(&sched_empty[slot]);
    if (++slot == TC_SQ) { slot = 0; sphase ^= 1; }
    if (it < 0) break;
    const TcItem I = p.items[it];
    const int buf = icount & 1;
    const int et = threadIdx.x;
    if (et < I.nq) {
      const int q = p.pair_query ? p.pair_query[I.pair_begin + et] : I.pair_begin + et;
      s_q[buf][et] = q;
      s_tau[buf][et] = MODE == 1 ? p.tau[q] : 0.f;
      if (HALF) s_qs[buf][et] = p.qscale[q];
    }
    asm volatile("bar.sync 1, %0;" ::"n"(C::CWARPS * 32) : "memory");
    const int hw = MODE == 1 ? warp : 0;
    auto consume = [&](auto n) {
      tc_consume_item<HALF, decltype(n)::value, C>(p, I, kblocks, sA, sB, full_bar, empty_bar, ring, s_tau[buf], s_q[buf], s_qs[buf],
                                                   s_hit_key[hw], s_hit_q[hw], &s_hit_n[hw]);
    };
    const int bl = tc_bcols_log(I.nq);
    if (bl == 0) consume(std::integral_constant<int, 16>());
    else if (bl == 1) consume(std::integral_constant<int, 32>());
    else if (MODE == 2 || bl == 2) consume(std::integral_constant<int, 64>());  // the dense form's groups stop at 64
    else if constexpr (MODE != 2) consume(std::integral_constant<int, 128>());
    if constexpr (MODE == 1) {  // flush this warp's staged hits
      __syncwarp();
      const int nh = min(s_hit_n[hw], TC_HITS);
      for (int i = lane; i < nh; i += 32) {
        const int q = s_hit_q[hw][i];
        const int sl = atomicAdd(p.cand_cnt + q, 1);
        if (sl < p.cap) p.cand[(size_t)q * p.cap + sl] = s_hit_key[hw][i];
      }
      __syncwarp();
      if (lane == 0) s_hit_n[hw] = 0;
      __syncwarp();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// per-query capture threshold T.  tau = the k-th smallest sampled score (TC_SAMPLE rows per span) bounds the k-th
// smallest score overall (A_k) from above; tc_tau_with_margin turns it into T.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float tc_eps(bool l2, float qnorm_sq, float max_norm, int d, int arith);

// Capture threshold from the sampled k-th score tau.  The finish kernel certifies A_k + 2 eps <= T (A_k = k-th captured
// score); a query that fails is re-run on the exact scan, and a single re-scanned query of a large shard stalls every rank
// of a sharded batch for milliseconds.  Two cases:
//   * at least TAU_SAFE sampled scores lie below tau - 2 eps: about TAU_SAFE * TC_SPAN / TC_SAMPLE rows do too, far more
//     than k, so A_k < tau - 2 eps almost surely (fewer than k such rows would have to produce TAU_SAFE sample hits at a
//     1 / 64 sampling rate: probability < 3e-4 even then) -> T = tau, the tightest capture set;
//   * otherwise the k-th row may sit within 2 eps of tau: capture under T = tau + 2 eps, which makes the certification true
//     by construction (A_k <= tau because the sample is a subset of the rows) at the price of a wider capture set — taken
//     only while the predicted number of captures leaves headroom in the capture buffer.
constexpr int TAU_SAFE = 3;
template <class CountLE>
__device__ __forceinline__ float tc_tau_with_margin(float tau, float two_eps, int cap, CountLE count_le) {
  if (count_le(__fsub_rd(tau, two_eps)) >= TAU_SAFE) return tau;
  const float lim = __fadd_ru(tau, two_eps);
  const float cs = (float)count_le(lim);  // sampled scores under T: the capture count is ~ (cs +- sqrt(cs)) * sampling ratio
  const float predicted = (cs + 4.f * sqrtf(cs)) * (float)(TC_SPAN / TC_SAMPLE);  // + 4 sigma: thousands of queries per batch
  return predicted <= (float)cap ? lim : tau;
}

constexpr int TAU_PL = 4096;  // (sample slot, column) pairs staged per query

// Block form of the threshold kernel, for the queries tc_tau_warp_kernel hands back (more sampled spans than a warp
// stages): one (sample slot, column) pair per sampled span, then the k-th smallest finite sampled score, selected by the
// whole CTA straight from the sample buffer.
static __global__ void __launch_bounds__(SCAN_THREADS)
tc_tau_kernel(const long long* __restrict__ probes, const int* __restrict__ pos, const int* __restrict__ cnt,
              const int* __restrict__ item_off, const int* __restrict__ list_len, const TcItem* __restrict__ items, int nprobe,
              const float* __restrict__ sample, int k, int l2, const float* __restrict__ qnorm, float max_norm, int d, int arith,
              int cand_cap, float* tau, const int* __restrict__ redo) {
  __shared__ int2 s_pairs[TAU_PL];
  __shared__ BlockSelShared S;
  __shared__ int s_np, s_cle;
  const int q = blockIdx.x;
  if (!redo[q]) return;  // finished by the warp kernel
  if (threadIdx.x == 0) s_np = 0;
  __syncthreads();
  for (int j = threadIdx.x; j < nprobe; j += blockDim.x) {
    const long long l = probes[(size_t)q * nprobe + j];
    if (l < 0) continue;
    const int len = list_len[l];
    if (len <= 0) continue;
    const int nc = (len + TC_CHUNK - 1) / TC_CHUNK, ng = (cnt[l] + TC_NQT - 1) / TC_NQT;
    const int ps = pos[(size_t)q * nprobe + j];
    const int g = ps / TC_NQT, n = ps % TC_NQT;
    const int nspan = (len + TC_SPAN - 1) / TC_SPAN;
    const int base = atomicAdd(&s_np, nspan);
    for (int sp = 0; sp < nspan; ++sp) {
      const int ch = sp * (TC_SPAN / TC_CHUNK);
      if (ch < nc && base + sp < TAU_PL) s_pairs[base + sp] = make_int2(items[item_off[l] + ch * ng + g].sample_slot, n);
    }
  }
  __syncthreads();
  const int np = s_np;
  // more sampled spans than the staging area holds: capture everything (overflow then falls back to the exact scan)
  if (np > TAU_PL) { if (threadIdx.x == 0) tau[q] = TC_INF; return; }
  const int tot = np * TC_SAMPLE;
  auto sampled = [&](int i) { const int2 pr = s_pairs[i / TC_SAMPLE]; return sample[((size_t)pr.x * TC_NQT + pr.y) * TC_SAMPLE + i % TC_SAMPLE]; };
  auto count_le = [&](float lim) {  // block-wide count of sampled scores <= lim (all threads call)
    __syncthreads();
    if (threadIdx.x == 0) s_cle = 0;
    __syncthreads();
    int c = 0;
    for (int i = threadIdx.x; i < tot; i += blockDim.x) c += sampled(i) <= lim ? 1 : 0;
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_cle, c);
    __syncthreads();
    return s_cle;
  };
  if (count_le(FLT_MAX) < k) { if (threadIdx.x == 0) tau[q] = TC_INF; return; }  // fewer than k finite sampled scores
  const float kth = ord2f(block_kth_key_any(k, S, [&](auto f) {
    for (int i = threadIdx.x; i < tot; i += blockDim.x) { const float v = sampled(i); if (v < TC_INF) f(f2ord(v)); }
  }));
  const float t = tc_tau_with_margin(kth, 2.f * tc_eps(l2 != 0, qnorm[q], max_norm, d, arith), cand_cap, count_le);
  if (threadIdx.x == 0) tau[q] = t;
}


// Warp-per-query form of the threshold kernel (the common case: <= WT_PAIRS sampled spans of TC_SAMPLE rows per query).
// Lanes walk the probe list, stage one (sample slot, column) per sampled span, then the warp reads one span per step
// (32 contiguous floats) and radix-selects the k-th smallest finite score.  Queries with more spans set redo[q] and are
// finished by tc_tau_kernel.
constexpr int WT_WARPS = 4;
constexpr int WT_PAIRS = 64;
static __global__ void __launch_bounds__(WT_WARPS * 32)
tc_tau_warp_kernel(const long long* __restrict__ probes, const int* __restrict__ pos, const int* __restrict__ cnt,
                   const int* __restrict__ item_off, const int* __restrict__ list_len, const TcItem* __restrict__ items, int nprobe,
                   const float* __restrict__ sample, int k, int nq, int l2, const float* __restrict__ qnorm, float max_norm, int d, int arith,
                   int cap, float* tau, int* redo) {
  __shared__ int s_hist[WT_WARPS][WS_BINS];
  __shared__ int s_pair[WT_WARPS][WT_PAIRS];
  __shared__ uint32_t s_val[WT_WARPS][WT_PAIRS * TC_SAMPLE];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = blockIdx.x * WT_WARPS + warp;
  if (q >= nq) return;
  int np = 0;
  for (int base = 0; base < nprobe; base += 32) {
    const int j = base + lane;
    int nspan = 0, first = 0, ng = 1, g = 0, n = 0;
    if (j < nprobe) {
      const long long l = probes[(size_t)q * nprobe + j];
      const int len = l >= 0 ? list_len[l] : 0;
      if (len > 0) {
        ng = (cnt[l] + TC_NQT - 1) / TC_NQT;
        const int ps = pos[(size_t)q * nprobe + j];
        g = ps / TC_NQT; n = ps % TC_NQT;
        nspan = (len + TC_SPAN - 1) / TC_SPAN;
        first = item_off[l];
      }
    }
    int incl = nspan;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    const int off = np + incl - nspan;
    for (int sp = 0; sp < nspan; ++sp)
      if (off + sp < WT_PAIRS) s_pair[warp][off + sp] = items[first + sp * (TC_SPAN / TC_CHUNK) * ng + g].sample_slot * TC_NQT + n;
    np += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (np > WT_PAIRS) { if (lane == 0) redo[q] = 1; return; }
  if (lane == 0) redo[q] = 0;
  __syncwarp();
  // one lane per sampled span: its 32 scores are one 128-byte line, fetched as 8 independent 16-byte loads, so the whole
  // query's sample is in flight at once (a warp-per-span loop would serialise one L2 round trip per span)
  __shared__ int s_nfin[WT_WARPS];
  if (lane == 0) s_nfin[warp] = 0;
  __syncwarp();
  for (int p = lane; p < np; p += 32) {
    const float4* src = reinterpret_cast<const float4*>(sample + (size_t)s_pair[warp][p] * TC_SAMPLE);
    float4 v[TC_SAMPLE / 4];
#pragma unroll
    for (int j = 0; j < TC_SAMPLE / 4; ++j) v[j] = src[j];
    const float* f = reinterpret_cast<const float*>(v);
    int c = 0;
#pragma unroll
    for (int j = 0; j < TC_SAMPLE; ++j) c += f[j] < TC_INF ? 1 : 0;
    int o = atomicAdd(&s_nfin[warp], c);
#pragma unroll
    for (int j = 0; j < TC_SAMPLE; ++j) if (f[j] < TC_INF) s_val[warp][o++] = f2ord(f[j]);
  }
  __syncwarp();
  const int nfin = s_nfin[warp];
  float t = TC_INF;
  if (nfin >= k) {
    int c_le;
    const uint32_t* vals = s_val[warp];
    t = ord2f(warp_kth_key(k, s_hist[warp], [&](auto f) { for (int i = lane; i < nfin; i += 32) f(vals[i]); }, c_le));
    t = tc_tau_with_margin(t, 2.f * tc_eps(l2 != 0, qnorm[q], max_norm, d, arith), cap,
                           [&](float lim) { int c = 0; for (int i = lane; i < nfin; i += 32) c += ord2f(vals[i]) <= lim ? 1 : 0; return __reduce_add_sync(0xffffffffu, c); });
  }
  if (lane == 0) tau[q] = t;
}

// ---------------------------------------------------------------------------------------------
// per query: window select on the approximate scores, exact rerank, certification
// ---------------------------------------------------------------------------------------------
constexpr int FIN_SEG = 2048;  // in-window rows staged per round

__device__ __forceinline__ float tc_eps(bool l2, float qnorm_sq, float max_norm, int d, int arith) {
  // rigorous bound on |approx score - exact score| (DESIGN.md 4.2).  Operand term (relative to ||q|| max ||x||):
  //   TF32 single pass: rows truncated (< 2^-10 relative) + query rounded to nearest (<= 2^-11) = 1.5 * 2^-10 (the 2^-21
  //     cross term and the FP32 accumulation are covered by the second summand);
  //   split pass (hi*hi + lo*hi + hi*lo): 2^-19;
  //   FP16: each operand vector is off by at most delta = 2^-11 + sqrt(d) 2^-39 of its norm (RN, plus underflow below the
  //     power-of-two scale), so the dot product by at most 2 delta + delta^2; the FP16 products are exact in FP32.
  // Accumulation term: FP32 sums of d terms on both sides (tensor core, norms, and the exact kernel itself).
  // Both terms are relative; below the normal range rounding errs by an absolute amount, which the underflow term covers:
  //   * the norms: a FP32 sum of d squares loses at most d * 2^-149 to underflow, so ||v|| <= sqrt(n2) + sqrt(d) 2^-74.5;
  //   * the tensor core may flush subnormal operands, products and partial sums: < 2^-126 per product and per add
  //     (at most 6d of them with the split pass, doubled by L2's 2 <q, x>), and < 2^-126 |partner| per flushed operand,
  //     so at most 2^-124 sqrt(d) (||q|| + ||x||) over the row (x 2 for hi and lo);
  //   * FP16: hscale * qscale underflows to 0 only below 2^-149, and then |<q, x>| < d 2^30 hscale qscale <= d 2^-119;
  //     a subnormal acc * (hscale * qscale) errs by <= 2^-150;
  //   * the exact FP32 sums on the CUDA cores round gradually: <= 2^-150 per operation.
  //   Together <= (d + 64) 2^-118 + sqrt(d) (||q|| + max ||x||) 2^-122.
  // Range: the bound is only returned while A (below) <= 2^125, so every norm, score, partial sum and exact distance stays
  // finite with room for the rounding; beyond it, or for a NaN norm, eps = +inf and the finish kernels hand the query to
  // the exact scan.
  const float qn = sqrtf(qnorm_sq) + sqrtf((float)d) * 0x1p-74f;
  max_norm += sqrtf((float)d) * 0x1p-74f;
  const float A = l2 ? (max_norm + qn) * (max_norm + qn) : qn * max_norm;
  if (!(A <= 0x1p125f)) return TC_INF;
  float rel = 0.0014648438f;  // 2^-10 + 2^-11
  if (arith == TC_ARITH_SPLIT) rel = 1.9073486e-6f;  // 2^-19
  else if (arith == TC_ARITH_FP16) {
    const float delta = __fadd_ru(4.8828125e-4f /*2^-11*/, __fmul_ru(sqrtf((float)d), 1.8189894e-12f /*2^-39*/));
    rel = __fmaf_ru(delta, delta, 2.f * delta);
  }
  const float operand = (l2 ? 2.f : 1.f) * rel * qn * max_norm;
  const float accum = 2.f * (float)(d + 64) * 5.9604645e-8f /*2^-24*/ * A;
  const float under = (float)(d + 64) * 0x1p-118f + sqrtf((float)d) * (qn + max_norm) * 0x1p-122f;
  return operand + accum + under;
}

// The window rows s_rows[0, m) re-scored exactly in the reference order by the block's NQUADS quads, one row per quad per
// round: s_kd[i] = ord(ranking score), s_id[i] = id_of(row).  The id is loaded before the distance so that the two overlap.
template <bool L2, int NQUADS, class IdOf>
__device__ __forceinline__ void tc_rescore_window(const int* s_rows, int m, const float* __restrict__ vecs, const float* qrow, int d,
                                                  bool vec, IdOf id_of, uint32_t* s_kd, long long* s_id) {
  const int quad = threadIdx.x >> 2, t = threadIdx.x & 3;
  for (int base = 0; base < m; base += NQUADS) {
    const int i = base + quad;
    const bool valid = i < m;
    const long long row = (long long)s_rows[valid ? i : 0];  // rows < 2^31
    const long long id = valid ? id_of(row) : -1;
    const float v = quad_distance<L2>(vecs + (size_t)row * d, qrow, d, t, vec);
    if (valid && t == 0) { s_kd[i] = f2ord(L2 ? v : -v); s_id[i] = id; }
  }
}

// ---------------------------------------------------------------------------------------------
// Finish kernel for the common case (at most HF_MAXW rows inside the 2*eps window): one 128-thread CTA per query.
// k-th approximate score A_k (block radix select), every captured row with score <= A_k + 2 eps re-scored exactly in the
// reference order, exact top-k by (distance, id), certification.  All 32 quads of the CTA re-score the window rows
// together (the ~40 random 3 KB row gathers per query are what this kernel waits on, so they are all issued at once) and a
// rank sort orders the exact pairs: 16 CTAs per SM.  Queries whose window is larger set redo[q] = 1 and are finished by
// tc_final_kernel.
// ---------------------------------------------------------------------------------------------
constexpr int HF_THREADS = 128;
constexpr int HF_STAGE = 512;   // captured keys staged in shared memory (the rest is re-read from global / L2 in every pass)
constexpr int HF_MAXW = 256;

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}

// RANGE: as tc_final_kernel's; the window is every captured row, and a query whose capture overflowed is handed straight to
// the exact scan (flags 2) without being re-scored.
template <bool L2, bool RANGE>
static __global__ void __launch_bounds__(HF_THREADS)
tc_final_hybrid_kernel(const unsigned long long* __restrict__ cand, const int* __restrict__ cand_cnt, int cap,
                       const float* __restrict__ tau, const float* __restrict__ qnorm, float max_norm, const float* __restrict__ q,
                       const float* __restrict__ vecs, const long long* __restrict__ ids, int d, int arith, int k,
                       float* out_dist, long long* out_ids, int* flags, int* redo, uint32_t thr_key, int raw_out, int* out_counts) {
  extern __shared__ __align__(16) unsigned char s_dyn[];  // the query row (d % 4 == 0)
  __shared__ BlockSelShared S;
  __shared__ unsigned long long s_keys[HF_STAGE];
  __shared__ int s_rows[HF_MAXW];
  __shared__ uint32_t s_kd[HF_MAXW];
  __shared__ long long s_id[HF_MAXW];
  __shared__ int s_m, s_hits;
  const int lane = threadIdx.x & 31;
  const int qi = blockIdx.x;
  const int total = cand_cnt[qi];
  if (RANGE && total > cap) {
    if (threadIdx.x == 0) { flags[qi] = 2; redo[qi] = 0; }
    return;
  }
  const int n = min(total, cap);
  const unsigned long long* c = cand + (size_t)qi * cap;
  const int nst = min(n, HF_STAGE);
  for (int i = threadIdx.x; i < (d >> 2); i += HF_THREADS) cp_async16(s_dyn + (size_t)i * 16, q + (size_t)qi * d + i * 4);
  for (int i = threadIdx.x; i < nst; i += HF_THREADS) s_keys[i] = c[i];
  if (threadIdx.x == 0) { s_m = 0; if (RANGE) s_hits = 0; }
  __syncthreads();
  auto key_at = [&](int i) -> unsigned long long { return i < nst ? s_keys[i] : c[i]; };
  float a_k = TC_INF;
  if (!RANGE && n >= k) a_k = ord2f(block_kth_key_any(k, S, [&](auto f) { for (int i = threadIdx.x; i < n; i += HF_THREADS) f((uint32_t)(key_at(i) >> 32)); }));
  const float two_eps = 2.f * tc_eps(L2, qnorm[qi], max_norm, d, arith);
  // outside the range eps covers (the scores may be inf or NaN; range: a threshold that is not finite): the exact scan re-runs it
  if (RANGE ? !(fabsf(tau[qi]) < TC_INF) : !(two_eps < TC_INF)) {
    cp_async_wait_all();      // the query row
    if (threadIdx.x == 0) { flags[qi] = 1; redo[qi] = 0; }
    return;
  }
  {
    const float window = a_k + two_eps;
    for (int base = 0; base < n; base += HF_THREADS) {
      const int i = base + threadIdx.x;
      unsigned long long e = 0;
      bool in = false;
      if (i < n) { e = key_at(i); in = RANGE || ord2f((uint32_t)(e >> 32)) <= window; }
      const unsigned msk = __ballot_sync(0xffffffffu, in);
      int wbase = 0;
      if (lane == 0 && msk) wbase = atomicAdd(&s_m, __popc(msk));
      wbase = __shfl_sync(0xffffffffu, wbase, 0);
      const int p = wbase + __popc(msk & ((1u << lane) - 1u));
      if (in && p < HF_MAXW) s_rows[p] = (int)(uint32_t)(e & 0xffffffffull);
    }
  }
  __syncthreads();
  const int m = s_m;
  if (m > HF_MAXW) { if (threadIdx.x == 0) redo[qi] = 1; return; }
  const float* qs = reinterpret_cast<const float*>(s_dyn);
  // every in-window row is prefetched towards L2 at once, then 32 quads score 32 rows per round straight from global memory
  // (no staging buffer: 16 CTAs per SM keep ~500 rows in flight per SM)
  const int lines = (d * 4 + 127) / 128;
  for (int i = threadIdx.x; i < m * lines; i += HF_THREADS) {
    const char* ptr = reinterpret_cast<const char*>(vecs + (size_t)(uint32_t)s_rows[i / lines] * d) + (size_t)(i % lines) * 128;
    asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr));
  }
  cp_async_wait_all();  // the query row
  __syncthreads();
  tc_rescore_window<L2, HF_THREADS / 4>(s_rows, m, vecs, qs, d, true, [&](long long row) { return ids[row]; }, s_kd, s_id);
  __syncthreads();
  int kept = k;
  if constexpr (RANGE) {  // rows outside the range become sentinels, which rank after every hit
    int h = 0;
    for (int i = threadIdx.x; i < m; i += HF_THREADS) {
      if (s_kd[i] < thr_key) ++h;
      else { s_kd[i] = KEY_SENTINEL_D; s_id[i] = KEY_SENTINEL_ID; }
    }
    h = __reduce_add_sync(0xffffffffu, h);
    if (lane == 0 && h) atomicAdd(&s_hits, h);
    __syncthreads();
    kept = min(s_hits, k);
  }
  block_rank_sort(s_kd, s_id, m, [&](int rank, int e) {
    if (rank < kept) {
      const float v = ord2f(s_kd[e]);
      const float raw = L2 ? v : -v;
      out_dist[(size_t)qi * k + rank] = (L2 || raw_out) ? raw : __fsub_rn(1.0f, raw);
      out_ids[(size_t)qi * k + rank] = s_id[e];
    }
  });
  for (int i = min(m, kept) + threadIdx.x; i < k; i += HF_THREADS) { out_dist[(size_t)qi * k + i] = 0.f; out_ids[(size_t)qi * k + i] = -1; }
  if (threadIdx.x == 0) {
    const float tq = tau[qi];
    flags[qi] = (total <= cap ? 0 : 2) | ((RANGE || tq == TC_INF || a_k + two_eps <= tq) ? 0 : 1);  // 1: threshold too tight, 2: capture overflow
    redo[qi] = 0;
    if (RANGE) out_counts[qi] = kept;
  }
}

// ---------------------------------------------------------------------------------------------
// Register-resident select (coarse finish): each of SEL_THREADS threads holds KPT <= 32 keys, so a query's whole score row
// lives in registers and the CTA needs only ~13 KB of shared memory (8 CTAs per SM hide each other's barriers).
// ---------------------------------------------------------------------------------------------
constexpr int SEL_THREADS = 256;
constexpr int SEL_MAX_ROWS = 32 * SEL_THREADS;  // score rows the register select holds
constexpr int SEL_WCAP = 512;    // window rows re-scored per query (more -> tc_coarse_final_kernel)

// Coarse finish: top-nprobe rows of one query's dense score row.
//   full mode (out_raw != NULL or ties at the k-th score): re-score every row within 2*eps of the k-th approximate score
//     exactly and emit them in exact (score, row) order.
//   set mode  (probe tables, whose order nobody reads): rows more than 2*eps below the k-th score are certainly among
//     the exact top-k (only the k - 1 rows below it can beat them), rows more than 2*eps above are certainly not; only the
//     few rows in between are re-scored to fill the remaining slots.
// flags[qi] = 1 when the window overflowed SEL_WCAP: tc_coarse_final_kernel then redoes that query.
template <bool L2, int KPT>
static __global__ void __launch_bounds__(SEL_THREADS)
tc_coarse_select_kernel(const float* __restrict__ dense, long long ld, int nrows, const float* __restrict__ qnorm, float max_norm,
                        const float* __restrict__ q, const float* __restrict__ vecs, int d, int k, long long id_offset, int api_scores,
                        long long* out_probes, float* out_raw, int* flags, const int* redo_in) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ BlockSelShared S;
  __shared__ int s_rows[SEL_WCAP];
  __shared__ uint32_t s_kd[SEL_WCAP];
  __shared__ long long s_id[SEL_WCAP];
  __shared__ int s_m, s_ns;
  const int qi = blockIdx.x;
  if (redo_in && !redo_in[qi]) { if (threadIdx.x == 0) flags[qi] = 0; return; }  // finished by the warp kernel
  float* qs = reinterpret_cast<float*>(smem);
  for (int i = threadIdx.x; i < d; i += SEL_THREADS) qs[i] = q[(size_t)qi * d + i];
  uint32_t key[KPT];
#pragma unroll
  for (int j = 0; j < KPT; ++j) {
    const int r = threadIdx.x + j * SEL_THREADS;
    key[j] = r < nrows ? f2ord(dense[(size_t)qi * ld + r]) : 0xFFFFFFFFu;
  }
  const uint32_t kth = block_kth_key_any(k, S, [&](auto f) {  // barriers inside: qs is visible afterwards
#pragma unroll
    for (int j = 0; j < KPT; ++j) if (key[j] != 0xFFFFFFFFu) f(key[j]);
  });
  const float a_k = ord2f(kth);
  const float two_eps = 2.f * tc_eps(L2, qnorm[qi], max_norm, d, TC_ARITH_SPLIT);
  const uint32_t thr_hi = f2ord(__fadd_ru(a_k, two_eps));
  const bool set_mode = out_raw == nullptr && S.c_le == k;
  const uint32_t thr_lo = f2ord(__fsub_rd(a_k, two_eps));
  if (threadIdx.x == 0) { s_m = 0; s_ns = 0; }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < KPT; ++j) {
    if (key[j] > thr_hi) continue;  // empty slots (0xFFFFFFFF) drop out here too
    const int r = threadIdx.x + j * SEL_THREADS;
    if (set_mode && key[j] <= thr_lo) out_probes[(size_t)qi * k + atomicAdd(&s_ns, 1)] = r + id_offset;
    else { const int pos = atomicAdd(&s_m, 1); if (pos < SEL_WCAP) s_rows[pos] = r; }
  }
  __syncthreads();
  const int m = s_m, ns = s_ns;
  // degenerate score row (many near-equal scores), or eps = +inf (NaN scores drop out of the window): redo on the
  // streaming kernel, which then re-scores every row
  if (m > SEL_WCAP || !(two_eps < TC_INF)) {
    if (threadIdx.x == 0) flags[qi] = 1;
    return;
  }
  if (threadIdx.x == 0) flags[qi] = 0;
  tc_rescore_window<L2, SEL_THREADS / 4>(s_rows, m, vecs, qs, d, (d & 3) == 0, [](long long row) { return row; }, s_kd, s_id);
  block_bitonic_sort(s_kd, s_id, m);  // pads to a power of two <= SEL_WCAP (itself one)
  const int need = k - ns;  // slots still open (set mode), all k otherwise
  for (int i = threadIdx.x; i < need; i += SEL_THREADS) {
    const bool have = i < m;
    out_probes[(size_t)qi * k + ns + i] = have ? s_id[i] + id_offset : -1;
    if (out_raw) {
      const float v = have ? ord2f(s_kd[i]) : 0.f;
      out_raw[(size_t)qi * k + i] = api_scores ? v : (L2 ? v : -v);
    }
  }
}


// Coarse finish for small centroid tables (nrows <= 32 * KPT <= 1024): one 128-thread CTA per query.  Warp 0 holds the
// score row in registers and does the selection (same full / set modes and +-2 eps rule as tc_coarse_select_kernel) with
// shuffles / ballots; all 32 quads then re-score the window rows together; a rank sort orders them.  Three block
// barriers.  Queries whose re-score window exceeds HC_MAXW rows set flags[qi] = 1 and go to tc_coarse_select_kernel.
constexpr int HC_THREADS = 128;
constexpr int HC_MAXW = 256;
template <bool L2, int KPT>
static __global__ void __launch_bounds__(HC_THREADS)
tc_coarse_select_hybrid_kernel(const float* __restrict__ dense, long long ld, int nrows, const float* __restrict__ qnorm, float max_norm,
                               const float* __restrict__ q, const float* __restrict__ vecs, int d, int k, long long id_offset, int api_scores,
                               long long* out_probes, float* out_raw, int* flags) {
  __shared__ int s_hist[WS_BINS];
  __shared__ int s_rows[HC_MAXW];
  __shared__ uint32_t s_kd[HC_MAXW];
  __shared__ long long s_id[HC_MAXW];
  __shared__ int s_m, s_ns;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qi = blockIdx.x;
  if (warp == 0) {
    uint32_t key[KPT];
#pragma unroll
    for (int j = 0; j < KPT; ++j) {
      const int r = lane + j * 32;
      key[j] = r < nrows ? f2ord(dense[(size_t)qi * ld + r]) : 0xFFFFFFFFu;
    }
    int c_le;
    const uint32_t kth = warp_kth_key(k, s_hist, [&](auto f) {
#pragma unroll
      for (int j = 0; j < KPT; ++j) if (key[j] != 0xFFFFFFFFu) f(key[j]);
    }, c_le);
    const float a_k = ord2f(kth);
    const float two_eps = 2.f * tc_eps(L2, qnorm[qi], max_norm, d, TC_ARITH_SPLIT);
    const uint32_t thr_hi = f2ord(__fadd_ru(a_k, two_eps));
    const uint32_t thr_lo = f2ord(__fsub_rd(a_k, two_eps));
    const bool set_mode = out_raw == nullptr && c_le == k;
    int ns = 0, m = 0;
#pragma unroll
    for (int j = 0; j < KPT; ++j) {
      const int r = lane + j * 32;
      const bool in = key[j] <= thr_hi && key[j] != 0xFFFFFFFFu;
      const bool sure = in && set_mode && key[j] <= thr_lo;
      const unsigned ms = __ballot_sync(0xffffffffu, sure), mw = __ballot_sync(0xffffffffu, in && !sure);
      const unsigned lt = (1u << lane) - 1u;
      if (sure) out_probes[(size_t)qi * k + ns + __popc(ms & lt)] = r + id_offset;
      if (in && !sure) { const int p = m + __popc(mw & lt); if (p < HC_MAXW) s_rows[p] = r; }
      ns += __popc(ms);
      m += __popc(mw);
    }
    if (lane == 0) { s_m = two_eps < TC_INF ? m : HC_MAXW + 1; s_ns = ns; }  // eps = +inf: as tc_coarse_select_kernel
  }
  __syncthreads();
  const int m = s_m, ns = s_ns;
  if (m > HC_MAXW) { if (threadIdx.x == 0) flags[qi] = 1; return; }  // (tc_coarse_select_kernel rewrites the whole output row)
  tc_rescore_window<L2, HC_THREADS / 4>(s_rows, m, vecs, q + (size_t)qi * d, d, (d & 3) == 0, [](long long row) { return row; }, s_kd, s_id);
  __syncthreads();
  const int need = k - ns;  // slots still open (set mode), all k otherwise
  block_rank_sort(s_kd, s_id, m, [&](int rank, int e) {
    if (rank < need) {
      out_probes[(size_t)qi * k + ns + rank] = s_id[e] + id_offset;
      if (out_raw) {
        const float v = ord2f(s_kd[e]);
        out_raw[(size_t)qi * k + rank] = api_scores ? v : (L2 ? v : -v);
      }
    }
  });
  for (int i = m + threadIdx.x; i < need; i += HC_THREADS) {
    out_probes[(size_t)qi * k + ns + i] = -1;
    if (out_raw) out_raw[(size_t)qi * k + i] = 0.f;
  }
  if (threadIdx.x == 0) flags[qi] = 0;
}

// Streaming window select, the fallback of both finishes (no limit on the number of keys or of window rows).  key_at(i),
// i < n, is (ord(approximate score) << 32 | row); id_of(row) is the id a row is reported under.  Pass 1: A_k = k-th
// smallest approximate score (+inf when n < k).  Pass 2: every row with score <= A_k + two_eps re-scored exactly in the
// reference order, FIN_SEG rows at a time, into `sel`, which ends holding the exact top-k by (distance, id).
// smem: tc_stream_smem(d, pool_cap) bytes.  Returns A_k + two_eps (NaN when two_eps = +inf: then pass 2 takes every row).
// RANGE: no pass 1; every row is re-scored and `sel` keeps the closest k whose exact key is below thr_key (the exact scan's
// range rule: its select starts from the threshold (thr_key, INT64_MIN)).  All SCAN_THREADS threads call.
static size_t tc_stream_smem(int d, int pool_cap) { return ((size_t)d * 4 + 15) / 16 * 16 + (size_t)FIN_SEG * 4 + BlockSelect::smem_bytes(pool_cap); }

template <bool L2, bool RANGE = false, class KeyAt, class IdOf>
__device__ __forceinline__ float tc_stream_window(BlockSelect& sel, unsigned char* smem, int pool_cap, const float* __restrict__ qrow,
                                                  const float* __restrict__ vecs, int d, int n, int k, float two_eps, KeyAt key_at,
                                                  IdOf id_of, uint32_t thr_key = 0) {
  __shared__ int s_m;
  float* qs = reinterpret_cast<float*>(smem);
  const size_t qbytes = ((size_t)d * 4 + 15) / 16 * 16;
  int* s_rows = reinterpret_cast<int*>(smem + qbytes);  // [FIN_SEG]
  unsigned char* pool = smem + qbytes + (size_t)FIN_SEG * 4;
  for (int i = threadIdx.x; i < d; i += blockDim.x) qs[i] = qrow[i];
  uint32_t wkey = 0xFFFFFFFFu;
  if constexpr (!RANGE) {
    sel.init(pool, pool_cap, k);
    // pass 1: k-th smallest approximate score
    for (int base = 0; base < n; base += blockDim.x) {
      sel.maybe_prune(blockDim.x);
      const int i = base + threadIdx.x;
      if (i < n) {
        const unsigned long long e = key_at(i);
        const uint32_t key = (uint32_t)(e >> 32);
        const long long row = (long long)(e & 0xffffffffull);
        if (sel.passes(key, row)) sel.push(key, row);
      }
    }
    sel.prune();
    const float a_k = *sel.count >= k ? ord2f(sel.kd[k - 1]) : TC_INF;
    __syncthreads();
    // window = A_k + two_eps (+inf when fewer than k rows) as a key; eps = +inf (outside the range it bounds): every row,
    // NaN scores included (a NaN fails every float comparison, but its key 0xFFFFFFFF is the largest)
    wkey = two_eps < TC_INF ? f2ord(a_k + two_eps) : 0xFFFFFFFFu;
  }
  // pass 2: exact distances (reference AVX-512 order) of every row inside the window
  sel.init(pool, pool_cap, k);
  if constexpr (RANGE) {
    if (threadIdx.x == 0) { *sel.thr_d = thr_key; *sel.thr_id = (long long)0x8000000000000000LL; }
    __syncthreads();
  }
  const int quad = threadIdx.x >> 2, t = threadIdx.x & 3;
  const bool vec = (d & 3) == 0;
  for (int seg = 0; seg < n; seg += FIN_SEG) {
    if (threadIdx.x == 0) s_m = 0;
    __syncthreads();
    const int e1 = min(n, seg + FIN_SEG);
    for (int i = seg + threadIdx.x; i < e1; i += blockDim.x) {
      const unsigned long long e = key_at(i);
      if ((uint32_t)(e >> 32) <= wkey) s_rows[atomicAdd(&s_m, 1)] = (int)(uint32_t)(e & 0xffffffffull);
    }
    __syncthreads();
    const int m = s_m;
    for (int base = 0; base < m; base += SCAN_QUADS) {
      sel.maybe_prune(SCAN_QUADS);
      const int i = base + quad;
      const bool valid = i < m;
      const uint32_t row = (uint32_t)s_rows[valid ? i : 0];
      const float v = quad_distance<L2>(vecs + (size_t)row * d, qs, d, t, vec);
      if (valid && t == 0) {
        const uint32_t key = f2ord(L2 ? v : -v);
        const long long id = id_of(row);
        if (sel.passes(key, id)) sel.push(key, id);
      }
    }
    __syncthreads();
  }
  sel.prune();
  return ord2f(wkey);
}

// RANGE (a range tc_search): tau holds the range capture threshold, not a sampled one; every captured row is re-scored and
// the closest k rows whose exact key is below thr_key are kept, as the exact scan keeps them, and out_counts holds the rows
// kept.  In either mode out_dist holds the raw metric value (L2 distance | ip) when raw_out, else the API distance.
template <bool L2, bool RANGE>
static __global__ void __launch_bounds__(SCAN_THREADS)
tc_final_kernel(const unsigned long long* __restrict__ cand, const int* __restrict__ cand_cnt, int cap,
                const float* __restrict__ tau, const float* __restrict__ qnorm, float max_norm, const float* __restrict__ q,
                const float* __restrict__ vecs, const long long* __restrict__ ids, int d, int arith, int k, int pool_cap,
                float* out_dist, long long* out_ids, int* flags, const int* redo, uint32_t thr_key, int raw_out, int* out_counts) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int qi = blockIdx.x;
  if (redo && !redo[qi]) return;  // finished by the hybrid kernel
  const float two_eps = 2.f * tc_eps(L2, qnorm[qi], max_norm, d, arith);
  // outside the range eps covers (range: a threshold that is not finite): the exact scan re-runs it
  if (RANGE ? !(fabsf(tau[qi]) < TC_INF) : !(two_eps < TC_INF)) { if (threadIdx.x == 0) flags[qi] = 1; return; }
  const int total = cand_cnt[qi];
  const unsigned long long* c = cand + (size_t)qi * cap;
  BlockSelect sel;
  const float window = tc_stream_window<L2, RANGE>(sel, smem, pool_cap, q + (size_t)qi * d, vecs, d, min(total, cap), k, two_eps,
                                                   [&](int i) { return c[i]; }, [&](uint32_t row) { return ids[row]; }, thr_key);
  const float tq = tau[qi];
  const bool certified = (total <= cap) && (RANGE || tq == TC_INF || window <= tq);
  const int have = *sel.count;
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    float api = 0.f;
    long long id = -1;
    if (i < have) {
      const float v = ord2f(sel.kd[i]);
      const float raw = L2 ? v : -v;
      api = (L2 || raw_out) ? raw : __fsub_rn(1.0f, raw);
      id = sel.kid[i];
    }
    out_dist[(size_t)qi * k + i] = api;
    out_ids[(size_t)qi * k + i] = id;
  }
  if (threadIdx.x == 0) {
    flags[qi] = certified ? 0 : 1;
    if (RANGE) out_counts[qi] = have;
  }
}

// coarse quantiser: every approximate score is available (dense row), so the window select is always certified
template <bool L2>
static __global__ void __launch_bounds__(SCAN_THREADS)
tc_coarse_final_kernel(const float* __restrict__ dense, long long ld, int nrows, const float* __restrict__ qnorm, float max_norm,
                       const float* __restrict__ q, const float* __restrict__ vecs, int d, int k, int pool_cap,
                       long long id_offset, int api_scores, long long* out_probes, float* out_raw, const int* redo) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int qi = blockIdx.x;
  if (redo && !redo[qi]) return;  // finished by the register select
  const float* row_scores = dense + (size_t)qi * ld;
  BlockSelect sel;
  tc_stream_window<L2>(sel, smem, pool_cap, q + (size_t)qi * d, vecs, d, nrows, k, 2.f * tc_eps(L2, qnorm[qi], max_norm, d, TC_ARITH_SPLIT),
                       [&](int i) { return ((unsigned long long)f2ord(row_scores[i]) << 32) | (unsigned)i; },
                       [](uint32_t row) { return (long long)row; });
  const int have = *sel.count;
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    out_probes[(size_t)qi * k + i] = i < have ? sel.kid[i] + id_offset : -1;
    if (out_raw) {
      const float v = i < have ? ord2f(sel.kd[i]) : 0.f;
      const float raw = L2 ? v : -v;
      out_raw[(size_t)qi * k + i] = api_scores ? v : raw;  // api_scores: the ranking score itself (L2 distance | -ip), ascending
    }
  }
}

static __global__ void tc_compact_flags_kernel(const int* __restrict__ flags, int nq, int* qmap, int* count) {
  __shared__ int s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  for (int base = 0; base < nq; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const int f = (i < nq) ? flags[i] : 0;
    if (f) qmap[atomicAdd(&s_cnt, 1)] = i;
  }
  __syncthreads();
  if (threadIdx.x == 0) *count = s_cnt;
}
void tc_compact_flags(const int* flags, int nq, int* qmap, int* count, cudaStream_t s) {
  tc_compact_flags_kernel<<<1, 1024, 0, s>>>(flags, nq, qmap, count);
}

static __global__ void max_norm_kernel(const float* __restrict__ n2, long long n, float* out) {
  float m = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) m = fmaxf(m, n2[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(out), __float_as_int(m));  // non-negative floats order as ints
}

float device_max_norm(IndexBase* ix, const float* norms_sq, int64_t n, cudaStream_t s) {
  if (n <= 0) return 0.f;
  float* d = ix->scratch.alloc<float>(1);
  B200VS_CUDA(cudaMemsetAsync(d, 0, 4, s));
  max_norm_kernel<<<(unsigned)std::min<int64_t>(1024, cdiv(n, 256)), 256, 0, s>>>(norms_sq, n, d);
  float h = 0.f;
  B200VS_CUDA(cudaMemcpyAsync(&h, d, 4, cudaMemcpyDeviceToHost, s));
  B200VS_CUDA(cudaStreamSynchronize(s));
  return std::sqrt(h);
}

static __global__ void row_norms_kernel(const float* __restrict__ x, long long n, int d, float* out) {
  const long long quad = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
  const int t = threadIdx.x & 3;
  const bool valid = quad < n;
  const float* row = x + (size_t)(valid ? quad : 0) * d;
  const float n2 = quad_distance<false>(row, row, d, t, (d & 3) == 0);
  if (valid && t == 0) out[quad] = n2;
}
void launch_row_norms(const float* x, int64_t n, int d, float* out, cudaStream_t s) {
  if (n <= 0) return;
  row_norms_kernel<<<(unsigned)cdiv(n * 4, 256), 256, 0, s>>>(x, n, d, out);
  B200VS_CUDA(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  B200VS_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres));
  if (!p || qres != cudaDriverEntryPointSuccess) fail(B200VS_EINTERNAL, "cuTensorMapEncodeTiled not available");
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// row-major matrix [rows, d] of floats (half = false) or halves; box = 128 B of K (32 floats / 64 halves) x box_rows,
// 128-byte swizzle
static CUtensorMap make_tmap(const void* base, int64_t rows, int d, int box_rows, bool half = false) {
  CUtensorMap m;
  cuuint64_t gdim[2] = {(cuuint64_t)d, (cuuint64_t)std::max<int64_t>(rows, 1)};
  cuuint64_t gstride[1] = {(cuuint64_t)d * (half ? 2 : 4)};
  cuuint32_t box[2] = {(cuuint32_t)(half ? 2 * TC_BK : TC_BK), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode()(&m, half ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim,
                            gstride, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) fail(B200VS_EINTERNAL, "cuTensorMapEncodeTiled failed: " + std::to_string((int)r));
  return m;
}

// A = the rows [a_rows, d] in a_box-row tiles (the form's TcCfg::BM), B = the query block [b_rows, d]; FP16 when half (the
// optional lo operands are always FP32)
static TcMaps make_tc_maps(const void* a, const float* a_lo, int64_t a_rows, int a_box, const void* b, const float* b_lo,
                           int64_t b_rows, int d, bool half) {
  TcMaps m;
  m.a = make_tmap(a, a_rows, d, a_box, half);
  m.a32 = make_tmap(a, a_rows, d, TC_SAMPLE, half);
  m.a_lo = a_lo ? make_tmap(a_lo, a_rows, d, a_box) : m.a;
  for (int i = 0; i < 4; ++i) {
    m.b[i] = make_tmap(b, b_rows, d, 16 << i, half);
    m.b_lo[i] = b_lo ? make_tmap(b_lo, b_rows, d, 16 << i) : m.b[i];
  }
  return m;
}

static int64_t tc_item_bound(const TcView& v, int64_t npairs) {
  return (npairs / TC_NQT + 1) * (int64_t)std::max(1, v.max_chunks_per_list) + v.total_chunks;
}
static int64_t tc_sample_bound(const TcView& v, int64_t npairs) {  // spans are 4 chunks: at most (chunks + 3) / 4 per list
  const int64_t max_spans = (v.max_chunks_per_list + 3) / 4 + 1;
  return (npairs / TC_NQT + 1) * max_spans + (v.total_chunks + 3) / 4 + v.nlist;
}
int tc_cand_cap(int k) { return std::min(16384, std::max(8192, next_pow2(256 * k))); }

// Per-device one-time setup: cudaFuncSetAttribute applies to the CURRENT device only, and one process may hold indexes
// on several GPUs (b200vs_params.device), so the opt-in shared-memory limits are raised once per device ordinal.
constexpr int TC_MAX_DEVICES = 64;
struct TcDevice {
  int sms = 0;
  int sample_ctas[2] = {0, 0};  // resident CTAs per SM of the sample form, [HALF]
  int dense_ctas[2] = {0, 0};   // ... and of the dense form
};
static std::mutex g_tc_init_mu;
static TcDevice g_tc_dev[TC_MAX_DEVICES];

// the sample and dense forms: several CTAs per SM
template <bool HALF, int MODE>
static int tc_ctas_per_sm() {
  using C = TcCfg<MODE>;
  auto* kernel = tc_scan_kernel<HALF, MODE>;
  B200VS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
  B200VS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
  int n = 0;
  B200VS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, C::THREADS, C::SMEM));
  if (getenv("B200VS_DEBUG_FLAGS"))
    fprintf(stderr, "[b200vs] tc %s kernel (%s): %d CTAs per SM\n", MODE == 0 ? "sample" : "dense", HALF ? "fp16" : "tf32", n);
  return std::max(1, n);
}

static TcDevice tc_init(int device) {
  if (device < 0 || device >= TC_MAX_DEVICES) fail(B200VS_EILLEGAL_PARAMETERS, "bad CUDA device ordinal");
  std::lock_guard<std::mutex> g(g_tc_init_mu);
  if (g_tc_dev[device].sms) return g_tc_dev[device];
  TcDevice dev;
  dev.sms = device_sm_count(device);
  B200VS_CUDA(cudaFuncSetAttribute(tc_scan_kernel<false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TcCfg<1>::SMEM));
  B200VS_CUDA(cudaFuncSetAttribute(tc_scan_kernel<true, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TcCfg<1>::SMEM));
  dev.sample_ctas[0] = tc_ctas_per_sm<false, 0>();
  dev.sample_ctas[1] = tc_ctas_per_sm<true, 0>();
  dev.dense_ctas[0] = tc_ctas_per_sm<false, 2>();
  dev.dense_ctas[1] = tc_ctas_per_sm<true, 2>();
  B200VS_CUDA(cudaFuncSetAttribute(tc_final_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));  // + static smem
  B200VS_CUDA(cudaFuncSetAttribute(tc_final_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));  // + static smem
  B200VS_CUDA(cudaFuncSetAttribute(tc_final_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));  // + static smem
  B200VS_CUDA(cudaFuncSetAttribute(tc_final_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));  // + static smem
  B200VS_CUDA(cudaFuncSetAttribute(tc_coarse_final_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));  // + static smem
  B200VS_CUDA(cudaFuncSetAttribute(tc_coarse_final_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));  // + static smem
  B200VS_CUDA(cudaFuncSetAttribute(tc_final_hybrid_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  B200VS_CUDA(cudaFuncSetAttribute(tc_final_hybrid_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  B200VS_CUDA(cudaFuncSetAttribute(tc_final_hybrid_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  B200VS_CUDA(cudaFuncSetAttribute(tc_final_hybrid_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  g_tc_dev[device] = dev;  // only after every attribute call succeeded
  return dev;
}

bool tc_eligible(const IndexBase* ix, const TcView& v, int64_t nq, int k, int nprobe, const SearchCtx& sc, bool range) {
  if (sc.exact_only) return false;
  if (ix->dim % 4 != 0 || ix->dim < 32) return false;      // TMA: 16-byte row pitch; tiny d is not worth a tile
  if (nq < 16 || k > (range ? 4096 : 128)) return false;   // tiny batches, wide k: exact scan; 4096 = the select's limit
  if (range && tc_stream_smem(ix->dim, select_pool_cap(k, SCAN_THREADS)) > 160 * 1024) return false;  // streaming finish
  if (!v.norms || !v.vecs) return false;
  if (!tc_norms_in_range(ix->metric == B200VS_L2, v.max_norm)) return false;
  return tc_plan_fits(v, nq, nprobe);
}

// tc_eps returns +inf once A > 2^125.  For L2, A = (||q|| + max ||x||)^2 >= max ||x||^2 for every query (rounding is
// monotone); for IP, A = ||q|| max ||x|| with ||q|| > 0 (tc_eps's underflow allowance), so an infinite max ||x|| makes
// every A infinite.  A NaN max ||x|| fails both tests.
bool tc_norms_in_range(bool l2, float max_norm) {
  return l2 ? max_norm * max_norm <= 0x1p125f : max_norm <= FLT_MAX;
}

bool tc_plan_fits(const TcView& v, int64_t nq, int nprobe) {
  if (v.arena_rows <= 0 || v.arena_rows >= (1LL << 31)) return false;
  const int64_t npairs = nq * nprobe;
  if (npairs >= (1LL << 30)) return false;
  if (tc_item_bound(v, npairs) >= (1LL << 28)) return false;
  if (tc_sample_bound(v, npairs) * TC_NQT * TC_SAMPLE * 4 > (4LL << 30)) return false;  // sample buffer too large (TC_SAMPLE rows per sampled item)
  return true;
}

// Queries rounded for one arithmetic, with ||q||^2 in norm: op = the TF32 (RN) rows, or the scaled FP16 rows with their
// power-of-two scales in scale; the split arithmetic also keeps the TF32 remainder in lo.
struct TcQueries {
  void* op;
  float *lo, *norm, *scale;
};

static TcQueries tc_round_queries(IndexBase* ix, TcArith arith, int64_t nq, const float* q, cudaStream_t s) {
  const int d = ix->dim;
  auto& S = ix->scratch;
  TcQueries r{};
  r.op = S.alloc<unsigned char>((size_t)nq * d * (arith == TC_ARITH_FP16 ? 2 : 4));
  if (arith == TC_ARITH_SPLIT) r.lo = S.alloc<float>((size_t)nq * d);
  r.norm = S.alloc<float>(nq);
  if (arith == TC_ARITH_FP16) r.scale = S.alloc<float>(nq);
  const unsigned grid = (unsigned)cdiv(nq * 32, 256);
  if (arith == TC_ARITH_SPLIT) tc_prep_queries_split_kernel<<<grid, 256, 0, s>>>(q, nq, d, static_cast<float*>(r.op), r.lo, r.norm);
  else if (arith == TC_ARITH_FP16) tc_prep_queries_half_kernel<<<grid, 256, 0, s>>>(q, nq, d, static_cast<__half*>(r.op), r.scale, r.norm);
  else tc_prep_queries_kernel<<<grid, 256, 0, s>>>(q, nq, d, static_cast<float*>(r.op), r.norm);
  B200VS_CUDA(cudaGetLastError());
  return r;
}

TcPairs tc_plan_pairs(IndexBase* ix, const TcView& v, int64_t nq, const long long* probes, int nprobe, const void* qrows,
                      int row_bytes, cudaStream_t s) {
  auto& S = ix->scratch;
  TcPairs P;
  P.npairs = nq * nprobe;
  P.bound = tc_item_bound(v, P.npairs);
  P.sbound = tc_sample_bound(v, P.npairs);
  P.cnt = S.alloc<int>(v.nlist);
  P.pos = S.alloc<int>(P.npairs);
  P.pair_off = S.alloc<int>(v.nlist);
  P.item_off = S.alloc<int>(v.nlist);
  P.totals = S.alloc<int>(4);
  P.work = S.alloc<int>(4);
  P.pair_query = S.alloc<int>(P.npairs);
  P.sample_list = S.alloc<int>(P.sbound);
  P.bws = S.alloc<unsigned char>((size_t)(P.npairs + TC_NQT) * row_bytes);
  P.items = S.alloc<TcItem>(P.bound);
  B200VS_CUDA(cudaMemsetAsync(P.cnt, 0, (size_t)v.nlist * 4, s));
  B200VS_CUDA(cudaMemsetAsync(P.work, 0, 16, s));
  tc_count_pairs_kernel<<<(unsigned)cdiv(P.npairs, 256), 256, 0, s>>>(probes, P.npairs, P.cnt, P.pos);
  tc_plan_kernel<<<1, 1024, 0, s>>>(P.cnt, v.list_len, v.nlist, P.pair_off, P.item_off, P.totals);
  tc_fill_pairs_kernel<<<(unsigned)cdiv(P.npairs * 32, 256), 256, 0, s>>>(probes, P.pos, P.pair_off, v.list_len, P.npairs, nprobe, row_bytes, qrows, P.pair_query, P.bws);
  tc_items_kernel<<<(unsigned)cdiv(v.nlist, 128), 128, 0, s>>>(P.cnt, v.list_len, P.pair_off, P.item_off, v.nlist, P.items, P.totals, P.sample_list);
  B200VS_CUDA(cudaGetLastError());
  ix->launch_count(4);
  return P;
}

// everything the float passes share: the pair plan, rounded queries, tensor maps
struct TcPlan : TcPairs {
  bool half;  // the FP16 mirror (v.vecs_h) instead of the FP32 rows
  TcQueries qry;
  TcMaps maps;
  TcDevice dev;
};

static TcPlan tc_prepare(IndexBase* ix, const TcView& v, int64_t nq, const float* q, const long long* probes, int nprobe, cudaStream_t s) {
  const int d = ix->dim;
  TcPlan P;
  P.dev = tc_init(ix->device);
  P.half = v.vecs_h != nullptr;
  const int esz = P.half ? 2 : 4;  // operand bytes per element
  P.qry = tc_round_queries(ix, P.half ? TC_ARITH_FP16 : TC_ARITH_TF32, nq, q, s);
  static_cast<TcPairs&>(P) = tc_plan_pairs(ix, v, nq, probes, nprobe, P.qry.op, d * esz, s);
  const void* rows = P.half ? static_cast<const void*>(v.vecs_h) : static_cast<const void*>(v.vecs);
  P.maps = make_tc_maps(rows, nullptr, v.arena_rows, TcCfg<1>::BM, P.bws, nullptr, P.npairs + TC_NQT, d, P.half);
  ix->launch_count(1);
  return P;
}

// The parameters both tile passes share; the caller sets the mode and what that mode reads and writes.
static TcParams tc_params(const TcView& v, int d, bool l2, const TcItem* items, const int* totals, const float* hscale,
                          const float* qscale) {
  TcParams p{};
  p.ids = v.ids; p.norms = v.norms; p.list_off = v.list_off; p.d = d; p.l2 = l2 ? 1 : 0;
  p.items = items; p.totals = totals; p.hscale = hscale; p.qscale = qscale;
  return p;
}

// One persistent launch of the tile kernel in the form of p.mode, at most one CTA per work item: the sample (mode 0) and
// dense (mode 2) forms with as many CTAs per SM as fit, the capture form (mode 1) one CTA per SM.  All CTAs draw items
// from the same work counter, so a loose work_bound (a host-side bound on the item count) costs no more than one empty
// claim per CTA.
template <int MODE>
static void tc_launch_form(int ctas_per_sm, const TcDevice& dev, bool half, int64_t work_bound, const TcMaps& maps, const TcParams& p,
                           cudaStream_t s) {
  const int grid = (int)std::min<int64_t>((int64_t)dev.sms * ctas_per_sm, std::max<int64_t>(1, work_bound));
  auto* kernel = half ? tc_scan_kernel<true, MODE> : tc_scan_kernel<false, MODE>;
  kernel<<<grid, TcCfg<MODE>::THREADS, TcCfg<MODE>::SMEM, s>>>(maps, p);
}
static void tc_launch(const TcDevice& dev, bool half, int64_t work_bound, const TcMaps& maps, const TcParams& p, cudaStream_t s) {
  const int h = half ? 1 : 0;
  if (p.mode == 0) tc_launch_form<0>(dev.sample_ctas[h], dev, half, work_bound, maps, p, s);
  else if (p.mode == 1) tc_launch_form<1>(1, dev, half, work_bound, maps, p, s);
  else tc_launch_form<2>(dev.dense_ctas[h], dev, half, work_bound, maps, p, s);
  B200VS_CUDA(cudaGetLastError());
}

// The exact scan over what a tile search covers (the probed lists, or the single list of a Flat view): the re-run of the
// queries the tile passes could not finish.
static ScanJob tc_exact_job(const TcView& v, bool l2, int d, const long long* probes, int nprobe, const SearchCtx& sc) {
  ScanJob job;
  job.l2 = l2; job.vecs = v.vecs; job.ids = v.ids; job.d = d; job.sc = &sc;
  if (!v.flat) {
    job.mode = 1; job.probes = probes; job.nprobe = nprobe; job.list_off = v.list_off; job.list_len = v.list_len;
    job.avg_candidates = v.nlist > 0 ? (double)v.arena_rows * nprobe / v.nlist : 0;
  }
  else { job.mode = 0; job.n = v.arena_rows; }
  return job;
}

// profiling counters of a tile search: [2] queries re-run on the exact scan, [6] work items of the capture pass,
// [7] the sum over items of (128-row tiles x padded query columns)
static void tc_profile_counts(IndexBase* ix, const int* qcount, const int* totals, cudaStream_t s) {
  int h = 0;
  B200VS_CUDA(cudaMemcpyAsync(&h, qcount, 4, cudaMemcpyDeviceToHost, s));
  B200VS_CUDA(cudaStreamSynchronize(s));
  ix->stats[2] = h;
  int t[4] = {0, 0, 0, 0};
  B200VS_CUDA(cudaMemcpyAsync(t, totals, 16, cudaMemcpyDeviceToHost, s));
  B200VS_CUDA(cudaStreamSynchronize(s));
  ix->stats[6] = t[0];
  ix->stats[7] = t[3];
}

// ---------------------------------------------------------------------------------------------
// range mode of the list scan: the capture threshold comes from the radius (DESIGN.md 4.6)
// ---------------------------------------------------------------------------------------------
// tau[q] = a bound on the tile score s~ of every row whose exact FP32 value passes the range test, rounded outwards:
//   L2: hit => D_fp32 <= thr, and |s~ - (D_fp32 - ||q||^2)| <= eps (tc_eps, which covers the exact kernel's own rounding)
//       with ||q||^2 the real norm, of which only the FP32 sum qnorm is known: ||q||^2 >= qnorm - (d + 64) 2^-24 qnorm -
//       d 2^-149, so s~ <= thr - (that) + eps;
//   IP / cosine: hit => -ip_fp32 <= -thr and |s~ + ip_fp32| <= eps, so s~ <= -thr + eps.
// NaN when eps or the threshold is not finite: the finish kernels hand such a query to the exact scan.
static __global__ void tc_range_tau_kernel(const float* __restrict__ qnorm, long long nq, int l2, float thr, float max_norm, int d,
                                           int arith, float* __restrict__ tau) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq) return;
  const float eps = tc_eps(l2 != 0, qnorm[i], max_norm, d, arith);
  float t;
  if (l2) {
    const float qerr = __fmaf_ru((float)(d + 64) * 5.9604645e-8f /*2^-24*/, qnorm[i], (float)d * 0x1p-149f);
    t = __fadd_ru(__fsub_ru(thr, __fsub_rd(qnorm[i], qerr)), eps);
  } else {
    t = __fadd_ru(-thr, eps);
  }
  tau[i] = (eps < TC_INF && fabsf(t) < TC_INF) ? t : __int_as_float(0x7fffffff);
}

void tc_search(IndexBase* ix, const TcView& v, const SearchReq& r, const float* q, const long long* probes, int nprobe, float thr_raw,
               cudaStream_t s) {
  const int d = ix->dim;
  const bool l2 = ix->metric == B200VS_L2;
  const int64_t nq = r.nq;
  const int k = r.k;
  const int cap = tc_cand_cap(k);
  const SearchCtx& sc = *r.sc;
  auto& S = ix->scratch;
  ix->phase(IndexBase::PH_PLAN, s);
  TcPlan P = tc_prepare(ix, v, nq, q, probes, nprobe, s);
  float* tau = S.alloc<float>(nq);
  unsigned long long* cand = S.alloc<unsigned long long>((size_t)nq * cap);
  int* cand_cnt = S.alloc<int>(nq);
  int* flags = S.alloc<int>(nq);
  int* redo = S.alloc<int>(nq);
  int* qmap = S.alloc<int>(nq);
  int* qcount = S.alloc<int>(1);
  B200VS_CUDA(cudaMemsetAsync(cand_cnt, 0, (size_t)nq * 4, s));

  TcParams p = tc_params(v, d, l2, P.items, P.totals, v.hscale, P.qry.scale);
  p.pair_query = P.pair_query;
  p.tau = tau; p.cand = cand; p.cand_cnt = cand_cnt; p.cap = cap;
  p.filt.has_range = sc.has_range; p.filt.negate = sc.negate; p.filt.rmin = sc.rmin; p.filt.rmax = sc.rmax;
  p.filt.sorted_ids = sc.sorted_ids_dev; p.filt.n_ids = sc.n_ids;
  const int pool = select_pool_cap(k, SCAN_THREADS);
  const int arith = P.half ? TC_ARITH_FP16 : TC_ARITH_TF32;

  // 1) per-query capture thresholds: from the radius, or from the sample pass
  if (r.range) {
    ix->phase(IndexBase::PH_TAU, s);
    tc_range_tau_kernel<<<(unsigned)cdiv(nq, 256), 256, 0, s>>>(P.qry.norm, nq, l2 ? 1 : 0, thr_raw, v.max_norm, d, arith, tau);
  } else {
    float* sample = S.alloc<float>((size_t)P.sbound * TC_NQT * TC_SAMPLE);
    p.sample_list = P.sample_list; p.sample = sample;
    p.mode = 0; p.work_counter = P.work;
    ix->phase(IndexBase::PH_SAMPLE, s);
    tc_launch(P.dev, P.half, P.sbound, P.maps, p, s);
    ix->phase(IndexBase::PH_TAU, s);
    // warp per query; the block kernel only redoes queries with more sampled spans than a warp stages
    tc_tau_warp_kernel<<<(unsigned)cdiv(nq, WT_WARPS), WT_WARPS * 32, 0, s>>>(probes, P.pos, P.cnt, P.item_off, v.list_len, P.items, nprobe, sample, k, (int)nq, l2 ? 1 : 0, P.qry.norm, v.max_norm, d, arith, cap, tau, redo);
    tc_tau_kernel<<<(unsigned)nq, SCAN_THREADS, 0, s>>>(probes, P.pos, P.cnt, P.item_off, v.list_len, P.items, nprobe, sample, k, l2 ? 1 : 0, P.qry.norm, v.max_norm, d, arith, cap, tau, redo);
    ix->launch_count(1);
  }
  // 2) capture pass: stream every probed list chunk once, keep rows under the threshold
  p.mode = 1; p.work_counter = P.work + 1;
  ix->phase(IndexBase::PH_CAPTURE, s);
  {
    ScopedKernelTimer timer(ix, s, ix->profiling);
    tc_launch(P.dev, P.half, P.bound, P.maps, p, s);
    timer.stop();
  }
  // 3) window select (top-k) or range test + exact rerank + certification
  ix->phase(IndexBase::PH_FINAL, s);
  const uint32_t thr_key = r.range ? f2ord(l2 ? thr_raw : -thr_raw) : 0u;
  const int raw = r.raw ? 1 : 0;
  float* od = r.od;
  long long* oi = r.oi;
  int* oc = r.range ? r.oc : nullptr;
  const int* fin_redo = nullptr;
  const size_t hsm = (size_t)d * 4;  // the query row
  if (hsm <= 96 * 1024) {  // block select + re-score; the streaming kernel below only redoes queries whose window exceeds HF_MAXW rows
    const auto hybrid = r.range ? (l2 ? tc_final_hybrid_kernel<true, true> : tc_final_hybrid_kernel<false, true>)
                                : (l2 ? tc_final_hybrid_kernel<true, false> : tc_final_hybrid_kernel<false, false>);
    hybrid<<<(unsigned)nq, HF_THREADS, hsm, s>>>(cand, cand_cnt, cap, tau, P.qry.norm, v.max_norm, q, v.vecs, v.ids, d, arith, k, od, oi, flags, redo, thr_key, raw, oc);
    fin_redo = redo;
    ix->launch_count(1);
  }
  const size_t fin_smem = tc_stream_smem(d, pool);
  const auto stream_fin = r.range ? (l2 ? tc_final_kernel<true, true> : tc_final_kernel<false, true>)
                                  : (l2 ? tc_final_kernel<true, false> : tc_final_kernel<false, false>);
  stream_fin<<<(unsigned)nq, SCAN_THREADS, fin_smem, s>>>(cand, cand_cnt, cap, tau, P.qry.norm, v.max_norm, q, v.vecs, v.ids, d, arith, k, pool, od, oi, flags, fin_redo, thr_key, raw, oc);
  tc_compact_flags(flags, (int)nq, qmap, qcount, s);
  B200VS_CUDA(cudaGetLastError());
  ix->launch_count(4);
  ix->stats[1] = nq;
  // 4) uncertified (top-k) or overflowed (range) queries re-run on the exact scan (device-side count: blocks beyond it
  //    exit immediately)
  ScanJob job = tc_exact_job(v, l2, d, probes, nprobe, sc);
  if (r.range) { job.has_thr = true; job.thr_raw = thr_raw; }
  ix->phase(IndexBase::PH_FALLBACK, s);
  run_scan_mapped(ix, job, nq, qmap, qcount, q, k, r.raw ? nullptr : od, r.raw ? od : nullptr, oi, oc, s);
  ix->phase(IndexBase::PH_OTHER, s);
  if (ix->profiling && getenv("B200VS_DEBUG_FLAGS")) {
    std::vector<int> hf(nq), hc(nq);
    std::vector<float> ht(nq);
    B200VS_CUDA(cudaMemcpyAsync(hf.data(), flags, (size_t)nq * 4, cudaMemcpyDeviceToHost, s));
    B200VS_CUDA(cudaMemcpyAsync(hc.data(), cand_cnt, (size_t)nq * 4, cudaMemcpyDeviceToHost, s));
    B200VS_CUDA(cudaMemcpyAsync(ht.data(), tau, (size_t)nq * 4, cudaMemcpyDeviceToHost, s));
    B200VS_CUDA(cudaStreamSynchronize(s));
    long long tot = 0; int mx = 0, r1 = 0, r2 = 0, ninf = 0;
    for (int64_t i = 0; i < nq; ++i) { tot += hc[i]; mx = std::max(mx, hc[i]); r1 += (hf[i] & 1); r2 += (hf[i] & 2) ? 1 : 0; ninf += std::isinf(ht[i]) ? 1 : 0; }
    fprintf(stderr, "[b200vs] tc_search nq=%lld cap=%d captured avg=%.1f max=%d flagged: threshold=%d overflow=%d tau_inf=%d\n", (long long)nq, cap, (double)tot / nq, mx, r1, r2, ninf);
    for (int64_t i = 0, shown = 0; i < nq && shown < 4; ++i) if (hf[i]) { fprintf(stderr, "[b200vs]   q=%lld flag=%d captured=%d tau=%g\n", (long long)i, hf[i], hc[i], ht[i]); ++shown; }
  }
  if (ix->profiling) tc_profile_counts(ix, qcount, P.totals, s);
}

bool tc_coarse_eligible(const IndexBase* ix, int64_t nq, int nrows, int nprobe) {
  if (ix->dim % 4 != 0 || ix->dim < 32) return false;
  if (nq < 16 || nrows < 64 || nprobe > 1024) return false;
  if (ix->dim > 8192) return false;  // the finish kernels keep the query row in (un-opted) dynamic shared memory
  if ((int64_t)nq * nrows * 4 > (1LL << 30)) return false;  // dense score matrix
  return true;
}

// One dense launch of the tile kernel (mode 2): dense[q * v.arena_rows + r] = approximate score of query q against row r
// (L2: ||x||^2 - 2 <q, x>; IP: -<q, x>; tombstoned rows +inf).  qr.lo == nullptr: single-pass TF32, qr.op holds the
// RN-rounded queries and the tensor core truncates the rows a_hi.  Otherwise the error-compensated split pass: the three
// products hi*hi + lo*hi + hi*lo accumulate into the same register accumulators (the lo operands ride in the next ring
// stage).  hscale != nullptr: qr.op and a_hi are scaled FP16 (the list scan's FP16 arithmetic), qr.scale / hscale their scales.
static void tc_dense_scan(IndexBase* ix, const TcView& v, bool l2, int64_t nq, const TcQueries& qr, const void* a_hi, const float* a_lo,
                          const float* hscale, float* dense, cudaStream_t s) {
  const TcDevice dev = tc_init(ix->device);
  const int d = ix->dim;
  const int nrows = (int)v.arena_rows;
  const bool half = hscale != nullptr;
  auto& S = ix->scratch;
  using C = TcCfg<2>;
  const int chunk = nrows <= 16384 ? C::BM : TC_CHUNK;  // small tables: one tile per item so the whole chip has work
  // Query-group width (the wgmma N): an item is bound by the tiles it moves from L2, not by its MMAs (DESIGN §4.2), and
  // every stage of it holds C::BM rows + w queries, so the launch takes about (waves of items over the CTA slots) x
  // (C::BM + w).  Take the widest group that minimises that product: at 1024 centroids x 1024 queries, 256 items of 64
  // queries fill 3 x 132 slots in one wave.  A score does not depend on the width or the tile: each element's K order is
  // the same.
  const int64_t slots = (int64_t)dev.sms * dev.dense_ctas[half ? 1 : 0];
  int nqt = TC_DENSE_NQT;
  int64_t best = INT64_MAX;
  for (int w = TC_DENSE_NQT; w >= 16; w >>= 1) {
    const int64_t cost = cdiv(cdiv(nrows, chunk) * cdiv(nq, w), slots) * (C::BM + w);
    if (cost < best) { best = cost; nqt = w; }
  }
  const int nitems = (int)(cdiv(nrows, chunk) * cdiv(nq, nqt));
  TcItem* items = S.alloc<TcItem>(nitems);
  int* totals = S.alloc<int>(4);
  int* work = S.alloc<int>(4);
  B200VS_CUDA(cudaMemsetAsync(work, 0, 16, s));
  tc_coarse_items_kernel<<<(unsigned)cdiv(nitems, 128), 128, 0, s>>>(nrows, (int)nq, chunk, nqt, items, totals);
  TcParams p = tc_params(v, d, l2, items, totals, hscale, qr.scale);
  p.mode = 2; p.dense = dense; p.dense_ld = nrows; p.work_counter = work; p.split = qr.lo != nullptr ? 1 : 0;
  const TcMaps maps = make_tc_maps(a_hi, a_lo, nrows, C::BM, qr.op, qr.lo, nq, d, half);
  ix->phase(IndexBase::PH_COARSE_SCAN, s);
  tc_launch(dev, half, nitems, maps, p, s);
}

// The register-select finish of the coarse pass, in its warp form (HYBRID: 32 threads hold the score row) or its block form
// (SEL_THREADS threads), at the smallest width KPT, 2 KPT, ..., 32 keys per thread that holds the row.
template <bool HYBRID, bool L2, int KPT>
static void tc_coarse_select(const TcView& v, int64_t nq, const float* dense, const float* qnorm, const float* q, int d, int k,
                             long long* out_probes, float* out_raw, int* flags, const int* redo_in, cudaStream_t s) {
  const int nrows = (int)v.arena_rows;
  if constexpr (KPT < 32) {
    if (nrows > (HYBRID ? 32 : SEL_THREADS) * KPT)
      return tc_coarse_select<HYBRID, L2, 2 * KPT>(v, nq, dense, qnorm, q, d, k, out_probes, out_raw, flags, redo_in, s);
  }
  const int api = v.api_scores ? 1 : 0;
  if constexpr (HYBRID)
    tc_coarse_select_hybrid_kernel<L2, KPT><<<(unsigned)nq, HC_THREADS, 0, s>>>(dense, nrows, nrows, qnorm, v.max_norm, q, v.vecs, d, k,
                                                                               v.id_offset, api, out_probes, out_raw, flags);
  else
    tc_coarse_select_kernel<L2, KPT><<<(unsigned)nq, SEL_THREADS, ((size_t)d * 4 + 15) / 16 * 16, s>>>(
        dense, nrows, nrows, qnorm, v.max_norm, q, v.vecs, d, k, v.id_offset, api, out_probes, out_raw, flags, redo_in);
}

// Coarse quantiser: ONE dense launch of the tile kernel in split mode (error-compensated TF32).  The operand error drops
// to 2^-19 relative, so the exact re-score window stays a few dozen rows even when all centroid distances are nearly
// equal (uniform high-dimensional data); what remains of eps is the FP32 accumulation term.
void tc_coarse(IndexBase* ix, const TcView& v, bool l2, int64_t nq, const float* q, int nprobe, long long* out_probes,
               float* out_raw, cudaStream_t s) {
  const int d = ix->dim;
  const int nrows = (int)v.arena_rows;
  auto& S = ix->scratch;
  ix->phase(IndexBase::PH_COARSE_PREP, s);
  const TcQueries qr = tc_round_queries(ix, TC_ARITH_SPLIT, nq, q, s);
  const float* qnorm = qr.norm;
  float* dense = S.alloc<float>((size_t)nq * nrows);
  tc_dense_scan(ix, v, l2, nq, qr, v.vecs_hi, v.vecs_lo, nullptr, dense, s);
  ix->phase(IndexBase::PH_COARSE_FINAL, s);
  const int pool = select_pool_cap(nprobe, SCAN_THREADS);
  const size_t fin_smem = tc_stream_smem(d, pool);
  if (fin_smem > 160 * 1024) fail(B200VS_EILLEGAL_PARAMETERS, "coarse quantiser: dimension / nprobe too large for one SM's shared memory");
  const int* fin_redo = nullptr;
  if (nrows <= SEL_MAX_ROWS && nprobe <= nrows) {
    // warp-select / block-re-score kernel for small tables, then the register-resident block select (8 CTAs per SM) for larger tables
    // and for the queries the warp kernel flagged, then the streaming kernel for what is still flagged (normally none)
    int* redo0 = S.alloc<int>(nq);
    int* redo = S.alloc<int>(nq);
    const int* redo_in = nullptr;
    if (nrows <= 1024 && 2 * nprobe <= HC_MAXW) {
      if (l2) tc_coarse_select<true, true, 8>(v, nq, dense, qnorm, q, d, nprobe, out_probes, out_raw, redo0, nullptr, s);
      else tc_coarse_select<true, false, 8>(v, nq, dense, qnorm, q, d, nprobe, out_probes, out_raw, redo0, nullptr, s);
      redo_in = redo0;
      ix->launch_count(1);
    }
    if (l2) tc_coarse_select<false, true, 4>(v, nq, dense, qnorm, q, d, nprobe, out_probes, out_raw, redo, redo_in, s);
    else tc_coarse_select<false, false, 4>(v, nq, dense, qnorm, q, d, nprobe, out_probes, out_raw, redo, redo_in, s);
    fin_redo = redo;
    ix->launch_count(1);
  }
  if (l2) tc_coarse_final_kernel<true><<<(unsigned)nq, SCAN_THREADS, fin_smem, s>>>(dense, nrows, nrows, qnorm, v.max_norm, q, v.vecs, d, nprobe, pool, v.id_offset, v.api_scores ? 1 : 0, out_probes, out_raw, fin_redo);
  else tc_coarse_final_kernel<false><<<(unsigned)nq, SCAN_THREADS, fin_smem, s>>>(dense, nrows, nrows, qnorm, v.max_norm, q, v.vecs, d, nprobe, pool, v.id_offset, v.api_scores ? 1 : 0, out_probes, out_raw, fin_redo);
  B200VS_CUDA(cudaGetLastError());
  ix->phase(IndexBase::PH_OTHER, s);
  ix->launch_count(4);
}

static __global__ void tc_eps_kernel(const float* __restrict__ qnorm, long long nq, int l2, float max_norm, int d, int arith, float* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nq) out[i] = tc_eps(l2 != 0, qnorm[i], max_norm, d, arith);
}

// Diagnostics: the sample pass's scores on a one-list (Flat) view, scattered to out [nq, nrows].  Query q sits in column
// pos[q] % TC_NQT of query group pos[q] / TC_NQT; span sp of the list is sampled by that group's item of chunk
// sp * TC_SPAN / TC_CHUNK (the lookup tc_tau_warp_kernel makes).  One thread per (query, span, sampled row).
static __global__ void tc_debug_sample_scores_kernel(const int* __restrict__ pos, const int* __restrict__ cnt,
                                                     const int* __restrict__ item_off, const TcItem* __restrict__ items,
                                                     const float* __restrict__ sample, long long nq, int nrows, float* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int nspan = (nrows + TC_SPAN - 1) / TC_SPAN;
  if (i >= nq * nspan * TC_SAMPLE) return;
  const int r = (int)(i % TC_SAMPLE), sp = (int)(i / TC_SAMPLE % nspan);
  const long long q = i / ((long long)TC_SAMPLE * nspan);
  const int row = sp * TC_SPAN + r;
  if (row >= nrows) return;
  const int ng = (cnt[0] + TC_NQT - 1) / TC_NQT, g = pos[q] / TC_NQT, n = pos[q] % TC_NQT;
  const int slot = items[item_off[0] + sp * (TC_SPAN / TC_CHUNK) * ng + g].sample_slot;
  out[(size_t)q * nrows + row] = sample[((size_t)slot * TC_NQT + n) * TC_SAMPLE + r];
}

void tc_debug_scores(IndexBase* ix, const TcView& v, bool l2, int64_t nq, const float* q, TcArith arith, bool sample,
                     float* out_scores, float* out_eps, cudaStream_t s) {
  const int d = ix->dim;
  auto& S = ix->scratch;
  const bool split = arith == TC_ARITH_SPLIT, half = arith == TC_ARITH_FP16;
  if (sample && (split || !v.flat)) fail(B200VS_EILLEGAL_PARAMETERS, "sample-pass scores exist for one-list views in the list-scan arithmetic");
  const TcQueries qr = tc_round_queries(ix, arith, nq, q, s);
  if (v.arena_rows > 0) {
    const void* a_hi = v.vecs;
    const float *a_lo = nullptr, *hscale = nullptr;
    if (split) {  // the same row split the IVF coarse quantiser keeps for its centroids
      float* hi = S.alloc<float>((size_t)v.arena_rows * d);
      float* lo = S.alloc<float>((size_t)v.arena_rows * d);
      launch_split_rows(v.vecs, v.arena_rows, d, hi, lo, s);
      a_hi = hi; a_lo = lo;
    } else if (half) {  // the same mirror an IVF-Flat index keeps for its lists
      __half* h = S.alloc<__half>((size_t)v.arena_rows * d);
      float* sc = S.alloc<float>(v.arena_rows);
      launch_half_rows(v.vecs, nullptr, v.arena_rows, d, h, sc, s);
      a_hi = h; hscale = sc;
    }
    if (!sample) {
      tc_dense_scan(ix, v, l2, nq, qr, a_hi, a_lo, hscale, out_scores, s);
    } else {  // the search's own planning and sample launch, every query probing the one list
      TcView sv = v;
      sv.vecs_h = half ? static_cast<const __half*>(a_hi) : nullptr;
      sv.hscale = hscale;
      long long* probes = S.alloc<long long>(nq);
      B200VS_CUDA(cudaMemsetAsync(probes, 0, (size_t)nq * 8, s));
      const TcPlan P = tc_prepare(ix, sv, nq, q, probes, 1, s);
      float* smp = S.alloc<float>((size_t)P.sbound * TC_NQT * TC_SAMPLE);
      TcParams p = tc_params(sv, d, l2, P.items, P.totals, sv.hscale, P.qry.scale);
      p.sample_list = P.sample_list; p.pair_query = P.pair_query; p.sample = smp;
      p.mode = 0; p.work_counter = P.work;
      tc_launch(P.dev, P.half, P.sbound, P.maps, p, s);
      B200VS_CUDA(cudaMemsetAsync(out_scores, 0xFF, (size_t)nq * v.arena_rows * 4, s));  // NaN: not sampled
      const int64_t n = nq * cdiv(v.arena_rows, TC_SPAN) * TC_SAMPLE;
      tc_debug_sample_scores_kernel<<<(unsigned)cdiv(n, 256), 256, 0, s>>>(P.pos, P.cnt, P.item_off, P.items, smp, nq, (int)v.arena_rows, out_scores);
    }
  }
  tc_eps_kernel<<<(unsigned)cdiv(nq, 256), 256, 0, s>>>(qr.norm, nq, l2 ? 1 : 0, v.max_norm, d, arith, out_eps);
  B200VS_CUDA(cudaGetLastError());
}

}  // namespace b200vs
