// ivf_pq.cu — IVF-PQ index: coarse quantiser + by-residual product quantiser, LUT scan on the GPU.
//
// Replaces faiss::IndexIVFPQ behind VectorIndexRawIvfPq (src/vector/vector_index_raw_ivf_pq.cc:551-571 Init,
// :457-500 Train, :157-210 Search) and the outer VectorIndexIvfPq switch between an inner Flat index and the
// real IVF-PQ (src/vector/vector_index_ivf_pq.cc:327-395: trained with fewer than
// max(256*nlist, 256*2^nbits) vectors -> Flat).
//
// Arithmetic (matches oracle/oracle_pq.cc so results are comparable bit for bit on a shared trained state):
//   encode : residual r = x - c[list]; per sub-space argmin_j ||r_m - cw[m][j]||^2, sequential un-fused sums,
//            first minimum wins.
//   IP     : dis = <q, c[list]> (hooked AVX-512 order) + sum_m sim[m][code_m],      sim[m][j] = <q_m, cw[m][j]>
//   L2     : dis = ||q - c[list]||^2 + sum_m (T[list][m][code_m] - 2 sim[m][code_m]), T = ||cw||^2 + 2 <c_m, cw>
//   LUT sums run sequentially over m in FP32.
// Codes: nbits in [1, 8], ksub = 2^nbits, faiss PQEncoderGeneric layout: a row is code_size = ceil(M*nbits/8) bytes and
//   code m occupies bits [m*nbits, (m+1)*nbits) of the row's little-endian bit stream (LSB first in each byte), pad bits
//   zero.  At nbits = 8 that is one byte per code.
// Kernels: pq_sim_kernel (per-query LUT), pq_precompute_kernel (T), pq_encode_kernel (+ pq_pack_kernel below 8 bits),
//   pq_scan_select_kernel (8 bits), pq_scan_packed_kernel<L2, NBITS> (1-7 bits).
#include <algorithm>
#include <memory>

#include "index.h"
#include "ivf_common.h"
#include "scan_kernels.cuh"

namespace b200vs {

IndexBase* make_flat(b200vs_metric m, int d, const b200vs_params& p);

namespace {

constexpr int KSUB = 256;       // the 8-bit scan kernel's LUT row
constexpr int PQ_THREADS = 512;  // code-scan CTA: one 96 KB LUT serves 16 warps (2 CTAs per SM -> 32 warps hide the code-load latency)
// packed-code scan CTA: the LUT is at most M * 128 floats (12 KB at M = 96, 4 bits), so shared memory no longer limits the
// CTAs per SM; 256 threads x 4 CTAs keep 32 warps resident within 64 registers (see DESIGN.md §4.3 for the ptxas figures)
constexpr int PQP_THREADS = 256;
constexpr int PQP_MIN_CTAS = 4;

__device__ __forceinline__ float ip_seq(const float* a, const float* b, int n) {
  float r = 0.f;
  for (int i = 0; i < n; ++i) r = __fadd_rn(r, __fmul_rn(a[i], b[i]));
  return r;
}

// sim[q][m][j] = <q_m, cw[m][j]>
__global__ void pq_sim_kernel(const float* __restrict__ q, const float* __restrict__ cb, long long nq, int d, int M, int ksub, float* sim) {
  const int dsub = d / M;
  const long long qi = blockIdx.x;
  const float* qv = q + (size_t)qi * d;
  for (int i = threadIdx.x; i < M * ksub; i += blockDim.x) {
    const int m = i / ksub;
    sim[(size_t)qi * M * ksub + i] = ip_seq(qv + m * dsub, cb + (size_t)i * dsub, dsub);
  }
}

// T[l][m][j] = ||cw||^2 + 2 <c_l,m , cw>
__global__ void pq_precompute_kernel(const float* __restrict__ cent, const float* __restrict__ cb, int d, int M, int ksub, float* pre) {
  const int dsub = d / M;
  const int l = blockIdx.x;
  for (int i = threadIdx.x; i < M * ksub; i += blockDim.x) {
    const int m = i / ksub;
    const float* cw = cb + (size_t)i * dsub;
    const float r2 = ip_seq(cw, cw, dsub);
    const float cr = ip_seq(cent + (size_t)l * d + m * dsub, cw, dsub);
    pre[(size_t)l * M * ksub + i] = __fadd_rn(r2, __fmul_rn(2.f, cr));
  }
}

// one warp per row: code[m] = argmin_j ||(x - c)_m - cw[m][j]||^2 over j < ksub, one byte per code
__global__ void pq_encode_kernel(const float* __restrict__ x, const long long* __restrict__ list, const float* __restrict__ cent,
                                 const float* __restrict__ cb, long long n, int d, int M, int ksub, unsigned char* codes_out) {
  extern __shared__ float s_res[];  // [warps_per_block][d]
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long w = (long long)blockIdx.x * (blockDim.x >> 5) + wib;
  if (w >= n) return;
  const int dsub = d / M;
  float* res = s_res + (size_t)wib * d;
  const float* xr = x + (size_t)w * d;
  const float* c = cent + (size_t)list[w] * d;
  for (int i = lane; i < d; i += 32) res[i] = __fsub_rn(xr[i], c[i]);
  __syncwarp();
  for (int m = 0; m < M; ++m) {
    const float* rs = res + m * dsub;
    float best = __int_as_float(0x7f800000);
    int bj = 0x7fffffff;
    for (int j = lane; j < ksub; j += 32) {  // lanes >= ksub keep (inf, INT_MAX) and never win the reduction
      const float* cw = cb + ((size_t)m * ksub + j) * dsub;
      float v = 0.f;
      for (int i = 0; i < dsub; ++i) { const float t = __fsub_rn(rs[i], cw[i]); v = __fadd_rn(v, __fmul_rn(t, t)); }
      if (v < best) { best = v; bj = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (ov < best || (ov == best && oj < bj)) { best = ov; bj = oj; }
    }
    if (lane == 0) codes_out[(size_t)w * M + m] = (unsigned char)bj;
  }
}

// byte-per-code rows [n, M] -> packed rows [n, cs]: one thread per output byte, pad bits zero
__global__ void pq_pack_kernel(const unsigned char* __restrict__ src, long long n, int M, int nbits, int cs, unsigned char* dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * cs) return;
  const long long r = i / cs;
  const int b0 = (int)(i % cs) * 8;
  const unsigned char* c = src + (size_t)r * M;
  unsigned v = 0;
  for (int t = 0; t < 8; ++t) {
    const int m = (b0 + t) / nbits;
    if (m < M) v |= ((c[m] >> ((b0 + t) % nbits)) & 1u) << t;
  }
  dst[i] = (unsigned char)v;
}

// rows of cs code bytes go to their slots
__global__ void scatter_codes_kernel(const unsigned char* __restrict__ src, const long long* __restrict__ src_ids,
                                     const long long* __restrict__ slots, long long n, int cs, unsigned char* codes, long long* ids) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * cs) return;
  const long long r = i / cs;
  const int m = (int)(i % cs);
  const long long s = slots[r];
  codes[(size_t)s * cs + m] = src[i];
  if (m == 0) ids[s] = src_ids[r];
}

__global__ void move_codes_kernel(const unsigned char* __restrict__ scodes, const long long* __restrict__ sids,
                                  const long long* __restrict__ src_rows, const long long* __restrict__ dst_rows, long long n, int cs,
                                  unsigned char* dcodes, long long* dids) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * cs) return;
  const long long r = i / cs;
  const int m = (int)(i % cs);
  dcodes[(size_t)dst_rows[r] * cs + m] = scodes[(size_t)src_rows[r] * cs + m];
  if (m == 0) dids[dst_rows[r]] = sids[src_rows[r]];
}

struct PqScanArgs {
  const unsigned char* codes;  // [rows, code_size]
  const long long* ids;
  const long long* probes;  // [nq, nprobe]
  const float* coarse;      // [nq, nprobe] raw metric value (ip or L2)
  const long long* list_off;
  const int* list_len;
  const float* sim;  // [nq, M*ksub]
  const float* pre;  // [nlist, M*ksub] (L2) or null
  int M, code_size, nprobe, k, nsplit, pool_cap;
  int has_thr;       // range search: fixed initial threshold (strict), k = max results kept
  uint32_t thr_key;
  uint32_t* ws_kd;
  long long* ws_kid;
  FilterDev filt;
};

// block (split, query): probes split round-robin; LUT in shared memory; one thread per code row.  Every eligible row goes to
// the sink (SelectSink, or DeepKeySink at its probe-prefix position).
template <bool L2, class Sink>
__device__ __forceinline__ void pq_scan_rows(const PqScanArgs& a, unsigned char* smem, const int qi, const int split, Sink& sink) {
  float* tab = reinterpret_cast<float*>(smem);
  const int M = a.M, T = M * KSUB;
  sink.init(smem + (size_t)T * 4);
  const float* simq = a.sim + (size_t)qi * T;
  if (!L2) {
    for (int i = threadIdx.x; i < T; i += blockDim.x) tab[i] = simq[i];
    __syncthreads();
  }
  for (int p = split; p < a.nprobe; p += a.nsplit) {
    const long long l = a.probes[(size_t)qi * a.nprobe + p];
    if (l < 0) continue;
    const int len = a.list_len[l];
    if (len <= 0) continue;
    const float dis0 = a.coarse[(size_t)qi * a.nprobe + p];
    if (L2) {  // fvec_madd(n, precomputed, -2, sim, tab)
      __syncthreads();
      const float* pl = a.pre + (size_t)l * T;
      for (int i = threadIdx.x; i < T; i += blockDim.x) tab[i] = __fadd_rn(pl[i], __fmul_rn(-2.0f, simq[i]));
      __syncthreads();
    }
    const long long base = a.list_off[l], pos0 = sink.list_pos(p);
    for (int r0 = 0; r0 < len; r0 += blockDim.x) {
      sink.step(blockDim.x);
      const int r = r0 + threadIdx.x;
      if (r < len) {
        const long long row = base + r;
        const long long id = a.ids[row];
        if (id >= 0 && filter_pass(a.filt, id)) {
          const unsigned char* code = a.codes + (size_t)row * M;
          float dis = dis0;
          if ((M & 15) == 0 && M <= 128) {
            // all code words of the row first (<= 8 independent 16-byte loads in flight), then the strictly ordered LUT sums
            uint4 cw[8];
#pragma unroll
            for (int g = 0; g < 8; ++g) if (g * 16 < M) cw[g] = *reinterpret_cast<const uint4*>(code + g * 16);
#pragma unroll
            for (int g = 0; g < 8; ++g) {
              if (g * 16 < M) {
                const uint32_t w[4] = {cw[g].x, cw[g].y, cw[g].z, cw[g].w};
#pragma unroll
                for (int j = 0; j < 16; ++j) dis = __fadd_rn(dis, tab[(g * 16 + j) * KSUB + ((w[j >> 2] >> (8 * (j & 3))) & 0xff)]);
              }
            }
          } else if ((M & 15) == 0) {
            for (int m0 = 0; m0 < M; m0 += 16) {
              const uint4 c = *reinterpret_cast<const uint4*>(code + m0);
              const uint32_t w[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
              for (int j = 0; j < 16; ++j) dis = __fadd_rn(dis, tab[(m0 + j) * KSUB + ((w[j >> 2] >> (8 * (j & 3))) & 0xff)]);
            }
          } else {
            for (int m = 0; m < M; ++m) dis = __fadd_rn(dis, tab[m * KSUB + code[m]]);
          }
          sink.take(f2ord(L2 ? dis : -dis), id, pos0 + r);
        }
      }
    }
  }
  sink.finish();
}
template <bool L2>
__global__ void __launch_bounds__(PQ_THREADS) pq_scan_select_kernel(const PqScanArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const size_t off = ((size_t)blockIdx.y * a.nsplit + blockIdx.x) * a.k;
  SelectSink sink(a.pool_cap, a.k, a.has_thr, a.thr_key, a.ws_kd + off, a.ws_kid + off);
  pq_scan_rows<L2>(a, smem, blockIdx.y, blockIdx.x, sink);
}
// deep top-k key pass: grid (nsplit, nqc), dynamic shared memory = the LUT
template <bool L2>
__global__ void __launch_bounds__(PQ_THREADS) pq_key_kernel(const PqScanArgs a, const DeepKeys o) {
  extern __shared__ __align__(16) unsigned char smem[];
  DeepKeySink sink(o, blockIdx.y);
  pq_scan_rows<L2>(a, smem, blockIdx.y, blockIdx.x, sink);
}


// Packed codes (NBITS < 8): 128 codes of a row take exactly 4*NBITS 32-bit words, so the row is read in chunks of
// 128 codes whose bit offsets are compile-time constants.  Chunk c of a row (words [4*NBITS*c, 4*NBITS*(c+1))) in the
// widest loads the row stride allows; words past the row's code_size bytes read as 0.
template <int NBITS>
__device__ __forceinline__ void pq_load_chunk(const unsigned char* code, int cs, int c, uint32_t (&w)[4 * NBITS]) {
  const int w0 = c * 4 * NBITS;
  if ((cs & 15) == 0) {  // rows 16-byte aligned
    const uint4* p = reinterpret_cast<const uint4*>(code);
    const int nv = cs >> 4;
#pragma unroll
    for (int i = 0; i < NBITS; ++i) {
      const uint4 v = c * NBITS + i < nv ? p[c * NBITS + i] : make_uint4(0u, 0u, 0u, 0u);
      w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w;
    }
  } else if ((cs & 3) == 0) {
    const uint32_t* p = reinterpret_cast<const uint32_t*>(code);
    const int nw = cs >> 2;
#pragma unroll
    for (int i = 0; i < 4 * NBITS; ++i) w[i] = w0 + i < nw ? p[w0 + i] : 0u;
  } else {
#pragma unroll
    for (int i = 0; i < 4 * NBITS; ++i) {
      uint32_t v = 0;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int o = (w0 + i) * 4 + b;
        if (o < cs) v |= (uint32_t)code[o] << (8 * b);
      }
      w[i] = v;
    }
  }
}

// dis += tab[j * ksub + code_j] for j = 0 .. n-1 of one chunk (n = 128, or the row's remaining codes when TAIL), in order.
// Code j sits at bit j*NBITS of the chunk: a shift of one word, or a funnel shift of two when it straddles a word boundary.
template <int NBITS, bool TAIL>
__device__ __forceinline__ float pq_sum_chunk(float dis, const float* tab, const uint32_t (&w)[4 * NBITS], int n) {
  constexpr int KS = 1 << NBITS;
#pragma unroll
  for (int j = 0; j < 128; ++j) {
    const int bit = j * NBITS, a = bit >> 5, s = bit & 31;
    const uint32_t v = s + NBITS <= 32 ? w[a] >> s : __funnelshift_r(w[a], w[a + 1], s);
    if (!TAIL || j < n) dis = __fadd_rn(dis, tab[j * KS + (v & (KS - 1))]);
  }
  return dis;
}

// The 8-bit kernel's scheme on packed rows: block (split, query), probes split round-robin, LUT [M, 2^NBITS] in shared
// memory (L2: rebuilt per probed list), one thread per code row, the same select and range-threshold epilogue.  A LUT
// row has at most 32 words, so the 32 lanes of a lookup touch 32 distinct banks at most: one wavefront per lookup.
template <bool L2, int NBITS, class Sink>
__device__ __forceinline__ void pq_scan_packed_rows(const PqScanArgs& a, unsigned char* smem, const int qi, const int split, Sink& sink) {
  constexpr int KS = 1 << NBITS;
  float* tab = reinterpret_cast<float*>(smem);
  const int M = a.M, T = M * KS, cs = a.code_size;
  sink.init(smem + (size_t)T * 4);
  const float* simq = a.sim + (size_t)qi * T;
  if (!L2) {
    for (int i = threadIdx.x; i < T; i += blockDim.x) tab[i] = simq[i];
    __syncthreads();
  }
  for (int p = split; p < a.nprobe; p += a.nsplit) {
    const long long l = a.probes[(size_t)qi * a.nprobe + p];
    if (l < 0) continue;
    const int len = a.list_len[l];
    if (len <= 0) continue;
    const float dis0 = a.coarse[(size_t)qi * a.nprobe + p];
    if (L2) {  // fvec_madd(n, precomputed, -2, sim, tab)
      __syncthreads();
      const float* pl = a.pre + (size_t)l * T;
      for (int i = threadIdx.x; i < T; i += blockDim.x) tab[i] = __fadd_rn(pl[i], __fmul_rn(-2.0f, simq[i]));
      __syncthreads();
    }
    const long long base = a.list_off[l], pos0 = sink.list_pos(p);
    for (int r0 = 0; r0 < len; r0 += blockDim.x) {
      sink.step(blockDim.x);
      const int r = r0 + threadIdx.x;
      if (r < len) {
        const long long row = base + r;
        const long long id = a.ids[row];
        if (id >= 0 && filter_pass(a.filt, id)) {
          const unsigned char* code = a.codes + (size_t)row * cs;
          float dis = dis0;
          uint32_t w[4 * NBITS];
          int c = 0;
          for (; (c + 1) * 128 <= M; ++c) {
            pq_load_chunk<NBITS>(code, cs, c, w);
            dis = pq_sum_chunk<NBITS, false>(dis, tab + c * 128 * KS, w, 128);
          }
          if (c * 128 < M) {
            pq_load_chunk<NBITS>(code, cs, c, w);
            dis = pq_sum_chunk<NBITS, true>(dis, tab + c * 128 * KS, w, M - c * 128);
          }
          sink.take(f2ord(L2 ? dis : -dis), id, pos0 + r);
        }
      }
    }
  }
  sink.finish();
}
template <bool L2, int NBITS>
__global__ void __launch_bounds__(PQP_THREADS, PQP_MIN_CTAS) pq_scan_packed_kernel(const PqScanArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const size_t off = ((size_t)blockIdx.y * a.nsplit + blockIdx.x) * a.k;
  SelectSink sink(a.pool_cap, a.k, a.has_thr, a.thr_key, a.ws_kd + off, a.ws_kid + off);
  pq_scan_packed_rows<L2, NBITS>(a, smem, blockIdx.y, blockIdx.x, sink);
}
template <bool L2, int NBITS>
__global__ void __launch_bounds__(PQP_THREADS, PQP_MIN_CTAS) pq_key_packed_kernel(const PqScanArgs a, const DeepKeys o) {
  extern __shared__ __align__(16) unsigned char smem[];
  DeepKeySink sink(o, blockIdx.y);
  pq_scan_packed_rows<L2, NBITS>(a, smem, blockIdx.y, blockIdx.x, sink);
}


// dis0[i] (i = query * nprobe + p) = the coarse pass's raw value (L2 distance or ip) of the query and list probes[i], for
// probes that come from the caller (a list-sharded search merges them from several ranks, and the ABI carries list ids
// only).  It is bit-equal to what the coarse pass of search hands the LUT scan: the exact scan's quad_distance on
// (centroid row, query), then its merge's (key, raw) round trip (which turns an ip of +0 into -0).  One quad per
// (query, probe); -1 probes and empty lists are skipped, as the LUT scans never read them.
template <bool L2>
__global__ void pq_dis0_kernel(const float* __restrict__ q, const float* __restrict__ cent, const long long* __restrict__ probes,
                               const int* __restrict__ list_len, long long n, int nprobe, int d, bool vec, float* dis0) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
  const int t = threadIdx.x & 3;
  const long long l = i < n ? probes[i] : -1;
  const bool valid = l >= 0 && list_len[l] > 0;
  // every quad of the warp takes part in quad_distance's shuffles: an idle quad evaluates query 0 against centroid 0
  const long long qi = valid ? i / nprobe : 0;
  const float v = quad_distance<L2>(cent + (size_t)(valid ? l : 0) * d, q + (size_t)qi * d, d, t, vec);
  if (valid && t == 0) dis0[i] = L2 ? ord2f(f2ord(v)) : -ord2f(f2ord(-v));
}

// the packed-code scan of NBITS = nbits: the top-k select, or the deep key pass into *keys when keys is set
template <bool L2>
void launch_pq_scan_packed(int nbits, dim3 grid, size_t smem, cudaStream_t s, const PqScanArgs& a, const DeepKeys* keys = nullptr) {
  auto go = [&](auto kern, auto key_kern) {
    if (keys) {
      B200VS_CUDA(cudaFuncSetAttribute(key_kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      key_kern<<<grid, PQP_THREADS, smem, s>>>(a, *keys);
      return;
    }
    B200VS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    kern<<<grid, PQP_THREADS, smem, s>>>(a);
  };
  switch (nbits) {
    case 1: go(pq_scan_packed_kernel<L2, 1>, pq_key_packed_kernel<L2, 1>); break;
    case 2: go(pq_scan_packed_kernel<L2, 2>, pq_key_packed_kernel<L2, 2>); break;
    case 3: go(pq_scan_packed_kernel<L2, 3>, pq_key_packed_kernel<L2, 3>); break;
    case 4: go(pq_scan_packed_kernel<L2, 4>, pq_key_packed_kernel<L2, 4>); break;
    case 5: go(pq_scan_packed_kernel<L2, 5>, pq_key_packed_kernel<L2, 5>); break;
    case 6: go(pq_scan_packed_kernel<L2, 6>, pq_key_packed_kernel<L2, 6>); break;
    case 7: go(pq_scan_packed_kernel<L2, 7>, pq_key_packed_kernel<L2, 7>); break;
    default: fail(B200VS_EINTERNAL, "no packed-code scan kernel for this nbits");
  }
}

}  // namespace

// Device rows of an IVF-PQ arena: [cap, cs] code bytes and ids (-1 = tombstone / unused slot).  The owner decides
// capacities and slots; the store moves rows.  All work runs on the owner's stream.
struct CodeRows {
  IndexBase* const ix;
  int cs = 0;  // bytes per packed code row (set by the owner)
  DevBuf<unsigned char> codes;
  DevBuf<long long> ids;
  explicit CodeRows(IndexBase* owner) : ix(owner) {}

  void grow(int64_t cap, int64_t keep) {
    codes.reserve((size_t)cap * cs, (size_t)keep * cs, ix->stream);
    ids.reserve(cap, keep, ix->stream);
  }
  void reset() { codes.free(); ids.free(); }
  void move(int64_t src, int64_t dst, int64_t n) {
    B200VS_CUDA(cudaMemcpyAsync(codes.p + (size_t)dst * cs, codes.p + (size_t)src * cs, (size_t)n * cs, cudaMemcpyDeviceToDevice, ix->stream));
    B200VS_CUDA(cudaMemcpyAsync(ids.p + dst, ids.p + src, (size_t)n * 8, cudaMemcpyDeviceToDevice, ix->stream));
  }
  // x / xids: device code rows and ids; row i goes to slot slots[i]
  void write(const unsigned char* x, const long long* xids, const std::vector<long long>& slots) {
    const int64_t n = (int64_t)slots.size();
    long long* d_slots = ix->scratch.alloc<long long>(n);
    B200VS_CUDA(cudaMemcpyAsync(d_slots, slots.data(), (size_t)n * 8, cudaMemcpyHostToDevice, ix->stream));
    scatter_codes_kernel<<<(unsigned)cdiv(n * cs, 256), 256, 0, ix->stream>>>(x, xids, d_slots, n, cs, codes.p, ids.p);
    B200VS_CUDA(cudaGetLastError());
  }
  // compaction: fresh buffers of cap rows holding row src[i] at dst[i]
  void gather(const std::vector<long long>& src, const std::vector<long long>& dst, int64_t cap) {
    const int64_t n = (int64_t)src.size();
    DevBuf<unsigned char> nc; DevBuf<long long> ni;
    nc.reserve((size_t)cap * cs, 0, ix->stream); ni.reserve(cap, 0, ix->stream);
    if (n) {
      long long* d_src = ix->scratch.alloc<long long>(n);
      long long* d_dst = ix->scratch.alloc<long long>(n);
      B200VS_CUDA(cudaMemcpyAsync(d_src, src.data(), n * 8, cudaMemcpyHostToDevice, ix->stream));
      B200VS_CUDA(cudaMemcpyAsync(d_dst, dst.data(), n * 8, cudaMemcpyHostToDevice, ix->stream));
      move_codes_kernel<<<(unsigned)cdiv(n * cs, 256), 256, 0, ix->stream>>>(codes.p, ids.p, d_src, d_dst, n, cs, nc.p, ni.p);
      B200VS_CUDA(cudaGetLastError());
    }
    B200VS_CUDA(cudaStreamSynchronize(ix->stream));
    codes.swap(nc); ids.swap(ni);
  }
  // rows [r0, r0 + n) as code rows [n, cs] on the host
  size_t row_bytes() const { return (size_t)cs; }
  void download(int64_t r0, int64_t n, uint8_t* out) const {
    if (n > 0) B200VS_CUDA(cudaMemcpy(out, codes.p + (size_t)r0 * cs, (size_t)n * cs, cudaMemcpyDeviceToHost));
  }
  const void* row_data() const { return codes.p; }
  size_t row_pitch() const { return (size_t)cs; }
  int64_t bytes() const { return (int64_t)(codes.cap + ids.cap * 8); }
};

struct IvfPqIndex : IndexBase {
  enum Mode { kNone, kFlat, kIvfPq } mode = kNone;
  int nlist, M, nbits;
  int ksub, code_size;              // 2^nbits codewords per sub-space; bytes per packed code row
  std::unique_ptr<IndexBase> flat;  // inner Flat index when there is too little data to train (ivf_pq.cc:339-353)
  DevBuf<float> centroids, codebooks, pre;
  DevBuf<long long> cent_ids;
  CodeRows store{this};             // the arena, [L.arena_cap] code rows
  IvfLists L;

  IvfPqIndex(b200vs_metric m, int d, const b200vs_params& p) : IndexBase(B200VS_IVF_PQ, m, d, p) {
    nlist = p.nlist > 0 ? p.nlist : 2048;      // Constant::kCreateIvfPqParamNcentroids
    M = p.pq_m > 0 ? p.pq_m : 64;              // kCreateIvfPqParamNsubvector
    nbits = p.pq_nbits > 0 ? p.pq_nbits : 8;   // kCreateIvfPqParamNbitsPerIdx
    if (nbits > 16) fail(B200VS_EILLEGAL_PARAMETERS, "nbits_per_idx must be in (0, 16]");
    if (nbits > 8)
      fail(B200VS_EILLEGAL_PARAMETERS, "nbits_per_idx 9-16 is not supported: the per-query LUT (M * 2^nbits floats) does not fit in "
                                       "shared memory, and the L2 precomputed table (nlist * M * 2^nbits floats) outgrows faiss's "
                                       "precomputed-table limit at realistic nlist");
    if (d % M != 0) fail(B200VS_EILLEGAL_PARAMETERS, "dimension must be divisible by nsubvector");
    ksub = 1 << nbits;
    code_size = (M * nbits + 7) / 8;
    store.cs = code_size;
  }
  bool is_trained() const override { return mode != kNone; }
  int sub_type() const override { return mode == kFlat ? (int)B200VS_FLAT : mode == kIvfPq ? (int)B200VS_IVF_PQ : -1; }  // ivf_pq.cc:474

  void install(const float* h_cent, const float* h_cb) {
    quiesce();
    centroids.free(); codebooks.free(); pre.free(); cent_ids.free();
    centroids.reserve((size_t)nlist * dim, 0, stream);
    codebooks.reserve((size_t)M * ksub * (dim / M), 0, stream);
    cent_ids.reserve(nlist, 0, stream);
    B200VS_CUDA(cudaMemcpyAsync(centroids.p, h_cent, (size_t)nlist * dim * 4, cudaMemcpyHostToDevice, stream));
    B200VS_CUDA(cudaMemcpyAsync(codebooks.p, h_cb, (size_t)M * ksub * (dim / M) * 4, cudaMemcpyHostToDevice, stream));
    launch_iota(cent_ids.p, nlist, stream);
    if (metric == B200VS_L2) {
      pre.reserve((size_t)nlist * M * ksub, 0, stream);
      pq_precompute_kernel<<<nlist, 256, 0, stream>>>(centroids.p, codebooks.p, dim, M, ksub, pre.p);
      B200VS_CUDA(cudaGetLastError());
    }
    B200VS_CUDA(cudaStreamSynchronize(stream));
    L.init(nlist, stream);
    store.reset();
    mode = kIvfPq;
  }

  // blob: int64 hdr[6] = {magic 'IVPQ', nlist, dim, metric, M, nbits}; centroids[nlist*dim]; codebooks[M*2^nbits*dsub]
  void set_state(const void* blob, size_t len) override {
    WriteHold hold(this);
    if (len < 48) fail(B200VS_EILLEGAL_PARAMETERS, "state blob too short");
    const int64_t* hdr = (const int64_t*)blob;
    if (hdr[0] != 0x51505649 || hdr[2] != dim || hdr[4] != M) fail(B200VS_EILLEGAL_PARAMETERS, "bad IVF-PQ state blob");
    if (hdr[5] != nbits) fail(B200VS_EILLEGAL_PARAMETERS, "IVF-PQ state blob has another nbits_per_idx than this index");
    nlist = (int)hdr[1];
    const size_t nc = (size_t)nlist * dim, ncb = (size_t)M * ksub * (dim / M);
    if (len < 48 + (nc + ncb) * 4) fail(B200VS_EILLEGAL_PARAMETERS, "state blob truncated");
    const float* f = (const float*)((const char*)blob + 48);
    install(f, f + nc);
  }
  int64_t get_state(void* blob, size_t cap) override {
    RwSharedGuard rl(this);
    if (mode != kIvfPq) return 0;
    const size_t nc = (size_t)nlist * dim, ncb = (size_t)M * ksub * (dim / M);
    const size_t need = 48 + (nc + ncb) * 4;
    if (!blob || cap < need) return (int64_t)need;
    set_device();
    int64_t hdr[6] = {0x51505649, nlist, dim, (int64_t)metric, M, nbits};
    memcpy(blob, hdr, 48);
    B200VS_CUDA(cudaMemcpyAsync((char*)blob + 48, centroids.p, nc * 4, cudaMemcpyDeviceToHost, stream));
    B200VS_CUDA(cudaMemcpyAsync((char*)blob + 48 + nc * 4, codebooks.p, ncb * 4, cudaMemcpyDeviceToHost, stream));
    B200VS_CUDA(cudaStreamSynchronize(stream));
    return (int64_t)need;
  }

  void assign_dev(const float* cd, int kk, const long long* cid, const float* x_dev, int dd, bool l2, int64_t n, long long* out,
                  cudaStream_t s) {
    ScanJob j;
    j.l2 = l2; j.vecs = cd; j.ids = cid; j.d = dd; j.mode = 0; j.n = kk;
    const int64_t chunk = 32768;
    for (int64_t a = 0; a < n; a += chunk) {
      const int64_t m = std::min(chunk, n - a);
      const auto mark = scratch.mark();
      run_scan(this, j, m, x_dev + (size_t)a * dd, 1, nullptr, nullptr, out + a, nullptr, s);
      scratch.release(mark);
    }
  }

  // VectorIndexIvfPq::Train (ivf_pq.cc:327-395) + VectorIndexRawIvfPq::Train (raw_ivf_pq.cc:457-500)
  void train(int64_t n, const void* xv) override {
    if (n <= 0) fail(B200VS_EILLEGAL_PARAMETERS, "data size invalid");
    WriteHold hold(this);
    if (mode != kNone) return;
    if (n < train_need()) {  // inner index = Flat
      flat.reset(make_flat(metric, dim, params));
      mode = kFlat;
      return;
    }
    const float* x = static_cast<const float*>(xv);
    std::vector<float> cent, cb;
    train_coarse_locked(n, x, nlist, cent);
    train_codebooks_locked(n, x, cent, cb);
    install(cent.data(), cb.data());
    train_rows = n;
  }
  int64_t train_need() const { return std::max<int64_t>(256LL * nlist, 256LL * ksub); }

  // VectorIndexIvfPq::NeedToRebuild (ivf_pq.cc:411-436): inner-Flat mode once train's `need` rows are held; IVF-PQ mode
  // VectorIndexRawIvfPq::NeedToRebuild (raw_ivf_pq.cc:518-526)
  bool need_rebuild() const override {
    if (mode == kFlat) {  // the inner index's writers hold its own lock only
      RwSharedGuard rl(flat.get());
      return flat->count() >= train_need();
    }
    if (mode == kIvfPq) return L.live / 2 >= train_rows;
    return false;
  }
  // a source in inner-Flat mode gives its inner index's rows; an IVF-PQ mode index keeps only codes: refused
  void live_rows(int64_t lo, int64_t hi, RebuildSource& out) override {
    if (mode == kIvfPq) fail(B200VS_EVECTOR_NOT_SUPPORT, "rebuild_from an IVF_PQ index in IVF-PQ mode: only its codes are stored");
    if (mode == kNone) return;
    out.hold = std::shared_lock<std::shared_mutex>(flat->rw);  // the inner index takes its writes under its own lock only
    flat->live_rows(lo, hi, out);
  }
  // from sources in inner-Flat mode: train's rule on their stored rows in ascending id order (IVF-PQ from `need` rows on,
  // else inner Flat again), then one add of them in that order
  int64_t rebuild_from(const std::vector<IndexBase*>& srcs, int64_t lo, int64_t hi) override {
    DevBuf<uint32_t> rows;
    DevBuf<long long> ids;
    const int64_t n = sorted_live_rows(this, srcs, lo, hi, dim, rows, ids, stream);
    if (n == 0) return 0;
    const float* x = reinterpret_cast<const float*>(rows.p);
    if (n < train_need()) {
      std::unique_ptr<IndexBase> f(make_flat(metric, dim, params));
      f->add(AddReq::device(n, x, ids.p, nullptr, false, AddReq::PREPARED));
      flat = std::move(f);
      mode = kFlat;
      train_rows = n;
      return n;
    }
    const int wpb = encode_warps();
    std::vector<float> cent, cb;
    train_coarse_locked(n, x, nlist, cent, true);
    train_codebooks_locked(n, x, cent, cb, true);
    install(cent.data(), cb.data());
    train_rows = n;
    scratch.reset(stream);
    add_locked(AddReq::device(n, x, ids.p, nullptr, false, AddReq::PREPARED), wpb);
    return n;
  }

  // The two stages of train, also run separately by the list-sharded trainer (shard.cu).  Callers take the writer hold.  x: raw host rows, or (x_dev) prepared rows on the device.  Coarse stage: k centroids of the n rows
  // (level-1 quantiser, niter 10).
  void train_coarse_locked(int64_t n, const float* x, int k, std::vector<float>& cent, bool x_dev = false) {
    const bool l2 = metric == B200VS_L2;
    DevBuf<long long> cid;
    auto assign = [&](const float* xd, int64_t m, const float* cd, int kk, long long* out) { assign_dev(cd, kk, cid.p, xd, dim, l2, m, out, stream); };
    auto prepare_ids = [&](int kk) { cid.free(); cid.reserve(kk, 0, stream); launch_iota(cid.p, kk, stream); };
    if (x_dev) kmeans_gpu_dev(this, dim, n, x, k, 10, 256, 1234, cent, assign, prepare_ids);
    else kmeans_gpu(this, metric, dim, n, x, k, 10, 256, 1234, cent, assign, prepare_ids);
  }

  // PQ stage: the codebooks [M, ksub, dsub] of the n rows' residuals to the centroids cent [nc, dim]
  void train_codebooks_locked(int64_t n, const float* x, const std::vector<float>& cent, std::vector<float>& cb, bool x_dev = false) {
    const bool l2 = metric == B200VS_L2;
    const int nc = (int)(cent.size() / dim);
    DevBuf<long long> cid;
    // PQ training set: <= 256 * ksub vectors (fvecs_maybe_subsample, seed 1234), residuals to their centroid
    int64_t m = std::min<int64_t>(n, 256LL * ksub);
    std::vector<int64_t> perm(n);
    for (int64_t i = 0; i < n; ++i) perm[i] = i;
    if (m < n) {
      std::mt19937 mt(1234);
      for (int64_t i = 0; i + 1 < n; ++i) { int64_t i2 = i + (int64_t)(mt() % (unsigned long)(n - i)); std::swap(perm[i], perm[i2]); }
    }
    std::vector<float> sub((size_t)m * dim);
    DevBuf<float> xd, cd;
    DevBuf<long long> asg, d_perm;
    xd.reserve((size_t)m * dim, 0, stream); cd.reserve((size_t)nc * dim, 0, stream); asg.reserve(m, 0, stream);
    if (x_dev) {  // the same sample, gathered on the device; the rows are already prepared
      d_perm.reserve(m, 0, stream);
      B200VS_CUDA(cudaMemcpyAsync(d_perm.p, perm.data(), (size_t)m * 8, cudaMemcpyHostToDevice, stream));
      launch_gather_words(reinterpret_cast<const uint32_t*>(x), d_perm.p, m, dim, reinterpret_cast<uint32_t*>(xd.p), stream);
    } else {
      for (int64_t i = 0; i < m; ++i) memcpy(&sub[(size_t)i * dim], x + (size_t)perm[i] * dim, (size_t)dim * 4);
      B200VS_CUDA(cudaMemcpyAsync(xd.p, sub.data(), (size_t)m * dim * 4, cudaMemcpyHostToDevice, stream));
      if (metric == B200VS_COSINE) launch_normalize_faiss(xd.p, m, dim, stream);
    }
    B200VS_CUDA(cudaMemcpyAsync(cd.p, cent.data(), (size_t)nc * dim * 4, cudaMemcpyHostToDevice, stream));
    cid.free(); cid.reserve(nc, 0, stream); launch_iota(cid.p, nc, stream);
    assign_dev(cd.p, nc, cid.p, xd.p, dim, l2, m, asg.p, stream);
    std::vector<long long> h_asg(m);
    B200VS_CUDA(cudaMemcpyAsync(h_asg.data(), asg.p, (size_t)m * 8, cudaMemcpyDeviceToHost, stream));
    B200VS_CUDA(cudaMemcpyAsync(sub.data(), xd.p, (size_t)m * dim * 4, cudaMemcpyDeviceToHost, stream));
    B200VS_CUDA(cudaStreamSynchronize(stream));
    for (int64_t i = 0; i < m; ++i) {
      const float* c = &cent[(size_t)h_asg[i] * dim];
      float* r = &sub[(size_t)i * dim];
      for (int j = 0; j < dim; ++j) r[j] -= c[j];
    }
    // one k-means per sub-space (ksub centroids, 25 iterations, L2)
    const int dsub = dim / M;
    std::vector<float> slice((size_t)m * dsub), cbm;
    cb.assign((size_t)M * ksub * dsub, 0.f);
    for (int mm = 0; mm < M; ++mm) {
      for (int64_t i = 0; i < m; ++i) memcpy(&slice[(size_t)i * dsub], &sub[(size_t)i * dim + mm * dsub], (size_t)dsub * 4);
      kmeans_gpu(this, B200VS_L2, dsub, m, slice.data(), ksub, 25, 256, 1234, cbm,
                 [&](const float* xs, int64_t mr, const float* cs, int kk, long long* out) { assign_dev(cs, kk, cid.p, xs, dsub, true, mr, out, stream); },
                 [&](int kk) { cid.free(); cid.reserve(kk, 0, stream); launch_iota(cid.p, kk, stream); });
      memcpy(&cb[(size_t)mm * ksub * dsub], cbm.data(), (size_t)ksub * dsub * 4);
    }
  }
  // the list-building calls (device write path, coarse slices, caller-supplied probes) need the IVF-PQ mode's lists
  void require_lists() const {
    if (mode == kFlat) fail(B200VS_EVECTOR_NOT_SUPPORT, "an IVF_PQ index in inner-Flat mode (too few training rows) has no inverted lists");
    if (mode == kNone) fail(B200VS_EVECTOR_NOT_TRAIN, "not train");
  }

  // warps per CTA of pq_encode_kernel: one residual row of shared memory per warp, 4 warps while they fit, fewer at large d
  // (opt-in above 48 KB).  Checked before anything changes.
  int encode_warps() const {
    constexpr size_t kEncodeSmemMax = 227 * 1024;
    const size_t row_bytes = (size_t)dim * 4;
    if (row_bytes > kEncodeSmemMax) fail(B200VS_EILLEGAL_PARAMETERS, "dimension too large for the PQ encoder's shared-memory residual");
    return (int)std::min<size_t>(4, kEncodeSmemMax / row_bytes);
  }
  // prepared rows st [n, dim] and their lists -> code rows [n, code_size] in the scratch (packed below 8 bits), on `stream`
  const unsigned char* encode_locked(int64_t n, const float* st, const long long* st_list, int wpb) {
    const size_t row_bytes = (size_t)dim * 4;
    unsigned char* st_codes = scratch.alloc<unsigned char>((size_t)n * M);
    B200VS_CUDA(cudaFuncSetAttribute(pq_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(wpb * row_bytes)));
    pq_encode_kernel<<<(unsigned)cdiv(n, wpb), wpb * 32, (size_t)wpb * row_bytes, stream>>>(st, st_list, centroids.p, codebooks.p, n, dim, M, ksub, st_codes);
    B200VS_CUDA(cudaGetLastError());
    if (nbits < 8) {
      unsigned char* packed = scratch.alloc<unsigned char>((size_t)n * code_size);
      pq_pack_kernel<<<(unsigned)cdiv(n * code_size, 256), 256, 0, stream>>>(st_codes, n, M, nbits, code_size, packed);
      B200VS_CUDA(cudaGetLastError());
      st_codes = packed;
    }
    return st_codes;
  }

  // Inner-Flat mode takes host rows only (the inner index has no inverted lists); otherwise the rows are normalised for cosine (RAW), assigned to
  // the caller's lists or the nearest ones, encoded and placed, or placed as given (ENCODED), so that codes, ids and list
  // layout do not depend on the route.  An upsert's placement first removes the rows holding its ids.
  void add(const AddReq& r) override {
    if (mode == kFlat && !r.on_device) { flat->add(r); return; }
    WriteHold hold(this);
    require_lists();
    add_locked(r, r.form == AddReq::ENCODED ? 0 : encode_warps());
  }
  // add with the writer hold taken; wpb = encode_warps()
  void add_locked(const AddReq& r, int wpb) {
    const bool encoded = r.form == AddReq::ENCODED, normalise = metric == B200VS_COSINE && r.form == AddReq::RAW;
    Staged st;
    stage(r, encoded ? (size_t)code_size : (size_t)dim * 4, normalise, st);
    const float* x = static_cast<const float*>(st.x);
    if (normalise) launch_normalize_faiss(static_cast<float*>(st.x), r.n, dim, stream);
    std::vector<long long> h_list;
    const long long* lists = IvfLists::row_lists(this, r.n, r.lists, h_list, [&](long long* out) {
      assign_dev(centroids.p, nlist, cent_ids.p, x, dim, metric == B200VS_L2, r.n, out, stream);
    });
    L.check_lists(r.n, h_list.data());  // before the encoder reads the lists' centroids
    const unsigned char* codes = encoded ? static_cast<const unsigned char*>(st.x) : encode_locked(r.n, x, lists, wpb);
    L.place(r.n, h_list.data(), st.ids, codes, st.ids_dev, store, r.upsert);
  }

  // b200vs_assign_device: nearest centroid of prepared rows, ties to the smaller list id (the host add's assignment)
  void assign_lists_dev(int64_t n, const void* x_dev, long long* out_lists_dev, cudaStream_t s) override {
    require_lists();
    assign_dev(centroids.p, nlist, cent_ids.p, static_cast<const float*>(x_dev), dim, metric == B200VS_L2, n, out_lists_dev, s);
  }

  void reserve_lists(const int64_t* rows_per_list, int n_lists) override {
    WriteHold hold(this);
    require_lists();
    L.reserve(rows_per_list, n_lists, store);
  }

  int64_t remove(int64_t n, const int64_t* del) override {
    if (mode == kFlat) { const int64_t r = flat->remove(n, del); return r == 0 ? -1 : r; }  // Flat semantics: unknown ids are OK
    WriteHold hold(this);
    if (mode == kNone) return -1;
    return L.remove(n, del, store);
  }

  // VectorIndexIvfPq::Search (ivf_pq.cc:159-163: untrained -> empty results) and VectorIndexRawIvfPq::Search / RangeSearch
  // (raw_ivf_pq.cc:160-278): faiss IndexIVFPQ::search / range_search on the codes; range radius -> 1 - radius for IP / cosine
  // (:229-232), L2 keeps dis < radius, IP keeps dis > radius: the same LUT scan with a threshold epilogue instead of the
  // k-th-best threshold.  A caller's probe table takes the place of the coarse pass, dis0 recomputed per (query, probe).
  void search(const SearchReq& r, cudaStream_t s) override {
    if (mode == kNone) { fill_empty(r, s); return; }
    if (mode == kFlat && !r.probes) {  // delegate to the inner Flat index, sharing this call's stream and scratch discipline
      std::shared_lock<std::shared_mutex> rl(flat->rw);
      LaneGuard lg(flat.get(), s);
      flat->search(r, s);  // (an id-list filter lives in the outer lane's scratch: same stream, still locked)
      if (!r.range) for (int i = 0; i < 8; ++i) stats[i] = flat->stats[i].load();
      return;
    }
    if (r.deep) lut_smem();
    else if (r.probes) check_probe_search(r.nq, r.k);
    else scan_smem(r.k);  // checked before anything is launched
    const float* q = queries(r, s);
    const int nprobe = r.probes ? r.nprobe : resolve_nprobe(*r.sc);
    const long long* probes = r.probes;
    float* dis0 = nullptr;
    if (!probes) {  // coarse quantiser: top-nprobe lists + raw coarse values
      long long* own = scratch.alloc<long long>((size_t)r.nq * nprobe);
      dis0 = scratch.alloc<float>((size_t)r.nq * nprobe);
      coarse_rows(r.nq, q, nprobe, 0, nlist, dis0, own, s);
      probes = own;
    }
    if (profiling) profile_probed(this, probes, r.nq * nprobe, nlist, L.d_len.p, s);
    if (r.deep) {
      scan_lists_deep(r.nq, q, r.k, *r.sc, probes, dis0 ? dis0 : probe_dis0(r.nq, q, probes, nprobe, s), nprobe, r.od, r.raw, r.oi, s);
      return;
    }
    scan_lists(r.nq, q, r.k, *r.sc, probes, dis0 ? dis0 : probe_dis0(r.nq, q, probes, nprobe, s), nprobe, r.range,
               ip_like() ? 1.0F - r.radius : r.radius, r.raw ? nullptr : r.od, r.oi, r.oc, s, r.raw ? r.od : nullptr);
  }

  // shared memory of the LUT scan's CTA (LUT + select pool), refused above one SM's 227 KB
  size_t scan_smem(int k) const {
    const int threads = nbits == 8 ? PQ_THREADS : PQP_THREADS;
    const size_t smem = (size_t)M * ksub * 4 + BlockSelect::smem_bytes(select_pool_cap(k, threads));
    if (smem > 227 * 1024) fail(B200VS_EILLEGAL_PARAMETERS, "nsubvector / topk too large for the shared-memory LUT");
    return smem;
  }
  // shared memory of the LUT alone (the deep key pass holds no select pool), refused above one SM's 227 KB
  size_t lut_smem() const {
    const size_t smem = (size_t)M * ksub * 4;
    if (smem > 227 * 1024) fail(B200VS_EILLEGAL_PARAMETERS, "nsubvector too large for the shared-memory LUT");
    return smem;
  }
  int resolve_nprobe(const SearchCtx& sc) const {
    const int nprobe = sc.nprobe > 0 ? sc.nprobe : 80;  // Constant::kSearchIvfPqParamNprobe, raw_ivf_pq.cc:170
    return std::min(nprobe, nlist);                      // raw_ivf_pq.cc:190
  }
  // the coarse quantiser of search over centroid rows [c0, c1): top-nprobe GLOBAL list ids, and the raw coarse values
  // (L2 distance or ip) when out_raw is set
  void coarse_rows(int64_t nq, const float* q, int nprobe, int c0, int c1, float* out_raw, long long* out_lists, cudaStream_t s) {
    ScanJob cj;
    cj.l2 = metric == B200VS_L2; cj.vecs = centroids.p + (size_t)c0 * dim; cj.ids = cent_ids.p + c0; cj.d = dim; cj.mode = 0; cj.n = c1 - c0;
    run_scan(this, cj, nq, q, nprobe, nullptr, out_raw, out_lists, nullptr, s);
  }

  // per-query LUT -> code scan + select of the probed lists -> merge.  q prepared; coarse = dis0 per (query, probe).  Range
  // mode (has_thr): keep hits strictly inside the raw threshold (L2: dis < thr; IP: dis > thr), at most k of them, closest
  // first; out_counts = hits per query.
  void scan_lists(int64_t nq, const float* q, int k, const SearchCtx& sc, const long long* probes, const float* coarse, int nprobe,
                  bool has_thr, float thr_raw, float* od, long long* oi, int* oc, cudaStream_t s, float* oraw = nullptr) {
    const int T = M * ksub;
    const int threads = nbits == 8 ? PQ_THREADS : PQP_THREADS;
    const int pool_cap = select_pool_cap(k, threads);
    const size_t smem = scan_smem(k);
    const bool l2 = metric == B200VS_L2;
    float* sim = scratch.alloc<float>((size_t)nq * T);
    pq_sim_kernel<<<(unsigned)nq, 256, 0, s>>>(q, codebooks.p, nq, dim, M, ksub, sim);
    PqScanArgs a;
    a.codes = store.codes.p; a.ids = store.ids.p; a.probes = probes; a.coarse = coarse; a.list_off = L.d_off.p; a.list_len = L.d_len.p;
    a.sim = sim; a.pre = l2 ? pre.p : nullptr; a.M = M; a.code_size = code_size; a.nprobe = nprobe; a.k = k;
    a.nsplit = (int)std::max<int64_t>(1, std::min<int64_t>(nprobe, (device_sm_count(device) * 2 + nq - 1) / nq));
    a.pool_cap = pool_cap;
    a.has_thr = has_thr ? 1 : 0;
    a.thr_key = has_thr ? f2ord(l2 ? thr_raw : -thr_raw) : 0;
    a.ws_kd = scratch.alloc<uint32_t>((size_t)nq * a.nsplit * k);
    a.ws_kid = scratch.alloc<long long>((size_t)nq * a.nsplit * k);
    a.filt.has_range = sc.has_range; a.filt.negate = sc.negate; a.filt.rmin = sc.rmin; a.filt.rmax = sc.rmax;
    a.filt.sorted_ids = sc.sorted_ids_dev; a.filt.n_ids = sc.n_ids;
    const size_t smem2 = BlockSelect::smem_bytes(a.pool_cap);
    dim3 grid(a.nsplit, (unsigned)nq);
    ScopedKernelTimer timer(this, s, profiling);
    if (nbits < 8) {
      if (l2) launch_pq_scan_packed<true>(nbits, grid, smem, s, a);
      else launch_pq_scan_packed<false>(nbits, grid, smem, s, a);
    } else if (l2) {
      B200VS_CUDA(cudaFuncSetAttribute(pq_scan_select_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      pq_scan_select_kernel<true><<<grid, PQ_THREADS, smem, s>>>(a);
    } else {
      B200VS_CUDA(cudaFuncSetAttribute(pq_scan_select_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      pq_scan_select_kernel<false><<<grid, PQ_THREADS, smem, s>>>(a);
    }
    timer.stop();
    if (l2) {
      B200VS_CUDA(cudaFuncSetAttribute(merge_select_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      merge_select_kernel<true><<<(unsigned)nq, SCAN_THREADS, smem2, s>>>(a.ws_kd, a.ws_kid, a.nsplit, k, a.pool_cap, od, oraw, oi, oc, nullptr, nullptr);
    } else {
      B200VS_CUDA(cudaFuncSetAttribute(merge_select_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      merge_select_kernel<false><<<(unsigned)nq, SCAN_THREADS, smem2, s>>>(a.ws_kd, a.ws_kid, a.nsplit, k, a.pool_cap, od, oraw, oi, oc, nullptr, nullptr);
    }
    B200VS_CUDA(cudaGetLastError());
    launch_count(3);
  }

  // deep top-k (run_deep) over the LUT scan: its key pass runs the scan kernels with DeepKeySink on every query chunk
  void scan_lists_deep(int64_t nq, const float* q, int k, const SearchCtx& sc, const long long* probes, const float* coarse, int nprobe,
                       float* od, bool raw, long long* oi, cudaStream_t s) {
    const int T = M * ksub;
    const size_t smem = lut_smem();
    const bool l2 = metric == B200VS_L2;
    float* sim = scratch.alloc<float>((size_t)nq * T);
    pq_sim_kernel<<<(unsigned)nq, 256, 0, s>>>(q, codebooks.p, nq, dim, M, ksub, sim);
    B200VS_CUDA(cudaGetLastError());
    launch_count(1);
    PqScanArgs base{};
    base.codes = store.codes.p; base.ids = store.ids.p; base.list_off = L.d_off.p; base.list_len = L.d_len.p;
    base.pre = l2 ? pre.p : nullptr; base.M = M; base.code_size = code_size; base.nprobe = nprobe;
    base.filt.has_range = sc.has_range; base.filt.negate = sc.negate; base.filt.rmin = sc.rmin; base.filt.rmax = sc.rmax;
    base.filt.sorted_ids = sc.sorted_ids_dev; base.filt.n_ids = sc.n_ids;
    DeepJob dj;
    dj.l2 = l2; dj.mode = 1; dj.ids = store.ids.p; dj.probes = probes; dj.nprobe = nprobe; dj.list_off = L.d_off.p; dj.list_len = L.d_len.p;
    const int sms = device_sm_count(device);
    run_deep(this, dj, nq, k, od, raw, oi, [&](int64_t q0, int nqc, const DeepKeys& o, cudaStream_t st) {
      PqScanArgs a = base;
      a.sim = sim + (size_t)q0 * T; a.probes = probes + (size_t)q0 * nprobe; a.coarse = coarse + (size_t)q0 * nprobe;
      a.nsplit = std::max(1, std::min(nprobe, sms * 4 / nqc));
      const dim3 grid(a.nsplit, nqc);
      if (nbits < 8) {
        if (l2) launch_pq_scan_packed<true>(nbits, grid, smem, st, a, &o);
        else launch_pq_scan_packed<false>(nbits, grid, smem, st, a, &o);
      } else if (l2) {
        B200VS_CUDA(cudaFuncSetAttribute(pq_key_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        pq_key_kernel<true><<<grid, PQ_THREADS, smem, st>>>(a, o);
      } else {
        B200VS_CUDA(cudaFuncSetAttribute(pq_key_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        pq_key_kernel<false><<<grid, PQ_THREADS, smem, st>>>(a, o);
      }
      B200VS_CUDA(cudaGetLastError());
      launch_count(1);
    }, s);
  }

  // ---- list-sharded building blocks (include/b200vs.h), in the IVF-PQ mode only ----
  int nlist_now() const override { return nlist; }
  int resolve_nprobe_api(const SearchCtx& sc) const override { return resolve_nprobe(sc); }
  void coarse(int64_t nq, const void* xv, bool prepared, int nprobe, int c0, int c1, float* out_score, long long* out_lists,
              cudaStream_t s) override {
    require_lists();
    if (c0 < 0 || c1 > nlist || c0 >= c1 || nprobe <= 0 || nprobe > c1 - c0) fail(B200VS_EILLEGAL_PARAMETERS, "bad centroid range / nprobe");
    const float* xq = static_cast<const float*>(xv);
    coarse_rows(nq, prepared ? xq : prepare_queries(nq, xq, s), nprobe, c0, c1, out_score, out_lists, s);
    if (out_score && metric != B200VS_L2) launch_negate(out_score, nq * nprobe, s);  // -> ascending ranking score
  }
  // refusals of a probe-driven search that depend on its arguments and the trained state only: a sharded search checks them
  // before its first collective
  void check_probe_search(int64_t nq, int k, bool deep = false) const override {
    require_lists();
    if (nq > 65535) fail(B200VS_EILLEGAL_PARAMETERS, "batch too large (max 65535 queries per call)");
    if (deep) lut_smem();
    else scan_smem(k);
  }
  // dis0 of every (query, probe) of a caller-supplied probe table
  const float* probe_dis0(int64_t nq, const float* q, const long long* probes, int nprobe, cudaStream_t s) {
    const long long n = (long long)nq * nprobe;
    float* dis0 = scratch.alloc<float>((size_t)n);
    const bool vec = (dim & 3) == 0 && (reinterpret_cast<uintptr_t>(q) & 15) == 0;  // the load width only, not the arithmetic
    const unsigned grid = (unsigned)cdiv(n * 4, 256);
    if (n <= 0) {
    } else if (metric == B200VS_L2) pq_dis0_kernel<true><<<grid, 256, 0, s>>>(q, centroids.p, probes, L.d_len.p, n, nprobe, dim, vec, dis0);
    else pq_dis0_kernel<false><<<grid, 256, 0, s>>>(q, centroids.p, probes, L.d_len.p, n, nprobe, dim, vec, dis0);
    B200VS_CUDA(cudaGetLastError());
    return dis0;
  }

  int64_t count() const override { return mode == kFlat ? flat->count() : L.live; }
  int64_t deleted_count() const override { return mode == kFlat ? flat->deleted_count() : L.dead; }
  int64_t memory_size() const override {
    if (mode == kFlat) return flat->memory_size();
    return store.bytes() + (int64_t)(centroids.cap * 4 + codebooks.cap * 4 + pre.cap * 4);  // raw_ivf_pq.cc:440-450
  }
  // Save / Load (reference: faiss::write_index / read_index of the IndexIVFPQ, vector_index_raw_ivf_pq.cc:298 and :314): own
  // container "B2VSPQ01" = mode, then either the inner Flat index's rows or {trained-state blob, list offsets, ids,
  // PQ codes in list-major order}.  Codes are restored as stored (never re-encoded: the vectors are gone).
  void save(const std::string& path) override {
    RwSharedGuard hold(this);  // one reader hold across count / trained state / export
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) fail(B200VS_EINTERNAL, "cannot open " + path);
    auto wr = [&](const void* p, size_t n) { if (n && fwrite(p, 1, n, f) != n) fail(B200VS_EINTERNAL, "short write"); };
    try {
      int64_t hdr[8] = {0, (int64_t)mode, (int64_t)metric, dim, nlist, M, 0, 0};
      memcpy(hdr, "B2VSPQ01", 8);
      if (mode == kFlat) {
        const int64_t n = flat->count();
        std::vector<int64_t> off(2, 0), fids((size_t)n);
        std::vector<float> vec((size_t)n * dim);
        if (n) flat->export_lists(off.data(), vec.data(), nullptr, fids.data());
        hdr[6] = n;
        wr(hdr, sizeof(hdr)); wr(fids.data(), fids.size() * 8); wr(vec.data(), vec.size() * 4);
      } else if (mode == kIvfPq) {
        const int64_t st_len = get_state(nullptr, 0);
        std::vector<unsigned char> st((size_t)st_len);
        get_state(st.data(), st.size());
        const int64_t n = count();
        std::vector<int64_t> off((size_t)nlist + 1, 0), fids((size_t)n);
        std::vector<uint8_t> cds((size_t)n * code_size);
        export_lists(off.data(), nullptr, cds.data(), fids.data());
        hdr[6] = n; hdr[7] = st_len;
        wr(hdr, sizeof(hdr)); wr(st.data(), st.size()); wr(off.data(), off.size() * 8); wr(fids.data(), fids.size() * 8); wr(cds.data(), cds.size());
      } else {
        wr(hdr, sizeof(hdr));  // untrained: nothing but the header
      }
    } catch (...) { fclose(f); throw; }
    fclose(f);
  }
  // save's bytes: the inner Flat index's rows, or the trained state and the code rows, packed on the device
  void save_image(SnapshotImage& img) override {
    RwSharedGuard hold(this);
    int64_t hdr[8] = {0, (int64_t)mode, (int64_t)metric, dim, nlist, M, 0, 0};
    memcpy(hdr, "B2VSPQ01", 8);
    if (mode == kFlat) {
      const int64_t n = flat->count();
      hdr[6] = n;
      img.alloc(sizeof(hdr) + (size_t)n * (8 + (size_t)dim * 4));
      int64_t off[2];
      if (n) flat->pack_lists(off, img.bytes.get() + sizeof(hdr), img.bytes.get() + sizeof(hdr) + (size_t)n * 8);
    } else if (mode == kIvfPq) {
      const int64_t st_len = get_state(nullptr, 0), n = count();
      hdr[6] = n; hdr[7] = st_len;
      const size_t off_at = sizeof(hdr) + (size_t)st_len, ids_at = off_at + ((size_t)nlist + 1) * 8, rows_at = ids_at + (size_t)n * 8;
      img.alloc(rows_at + (size_t)n * code_size);
      get_state(img.bytes.get() + sizeof(hdr), (size_t)st_len);
      std::vector<int64_t> off((size_t)nlist + 1, 0);
      if (n) pack_lists(off.data(), img.bytes.get() + ids_at, img.bytes.get() + rows_at);
      memcpy(img.bytes.get() + off_at, off.data(), off.size() * 8);
    } else {
      img.alloc(sizeof(hdr));  // untrained: nothing but the header
    }
    memcpy(img.bytes.get(), hdr, sizeof(hdr));
  }
  void load(const std::string& path) override {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) fail(B200VS_EINTERNAL, "cannot open " + path);
    auto rd = [&](void* p, size_t n) { if (n && fread(p, 1, n, f) != n) fail(B200VS_EINTERNAL, "short read / truncated index file"); };
    try {
      int64_t hdr[8];
      rd(hdr, sizeof(hdr));
      if (memcmp(hdr, "B2VSPQ01", 8) != 0 || hdr[2] != (int64_t)metric || hdr[3] != dim || hdr[5] != M)
        fail(B200VS_EINTERNAL, "index file does not match this index (type / metric / dimension / nsubvector)");
      if (mode != kNone) fail(B200VS_EINTERNAL, "load into a trained index");
      const int64_t n = hdr[6];
      if (hdr[1] == kFlat) {
        std::vector<int64_t> fids((size_t)n);
        std::vector<float> vec((size_t)n * dim);
        rd(fids.data(), fids.size() * 8); rd(vec.data(), vec.size() * 4);
        { std::unique_lock<std::shared_mutex> wl(rw); flat.reset(make_flat(metric, dim, params)); mode = kFlat; }
        for (int64_t a = 0; a < n; a += 32768)  // the rows come back exactly as stored
          flat->add(AddReq::host(std::min<int64_t>(32768, n - a), vec.data() + (size_t)a * dim, fids.data() + a, false, AddReq::PREPARED));
      } else if (hdr[1] == kIvfPq) {
        std::vector<unsigned char> st((size_t)hdr[7]);
        rd(st.data(), st.size());
        if (st.size() < 48 || ((const int64_t*)st.data())[5] != nbits)  // nbits travels in the embedded trained-state blob
          fail(B200VS_EINTERNAL, "index file does not match this index (nbits_per_idx)");
        set_state(st.data(), st.size());  // centroids, codebooks, precomputed table; nlist from the blob
        std::vector<int64_t> off((size_t)nlist + 1), fids((size_t)n);
        std::vector<uint8_t> cds((size_t)n * code_size);
        rd(off.data(), off.size() * 8); rd(fids.data(), fids.size() * 8); rd(cds.data(), cds.size());
        if (off[nlist] != n) fail(B200VS_EINTERNAL, "corrupt index file (list offsets)");
        WriteHold hold(this);
        std::vector<long long> h_list((size_t)n);
        for (int l = 0; l < nlist; ++l) for (int64_t i = off[l]; i < off[l + 1]; ++i) h_list[(size_t)i] = l;
        for (int64_t a = 0; a < n; a += 262144) {
          const int64_t m = std::min<int64_t>(262144, n - a);
          scratch.reset(stream);
          unsigned char* d_codes = scratch.alloc<unsigned char>((size_t)m * code_size);
          long long* d_ids = scratch.alloc<long long>(m);
          B200VS_CUDA(cudaMemcpyAsync(d_codes, cds.data() + (size_t)a * code_size, (size_t)m * code_size, cudaMemcpyHostToDevice, stream));
          B200VS_CUDA(cudaMemcpyAsync(d_ids, fids.data() + a, (size_t)m * 8, cudaMemcpyHostToDevice, stream));
          L.place(m, h_list.data() + a, fids.data() + a, d_codes, d_ids, store);
        }
      }
    } catch (...) { fclose(f); throw; }
    fclose(f);
  }

  void export_lists(int64_t* list_off, float* vectors, uint8_t* out_codes, int64_t* out_ids) override {
    if (mode == kFlat) { flat->export_lists(list_off, vectors, out_codes, out_ids); return; }
    RwSharedGuard rl(this);
    std::lock_guard<std::mutex> gl(gpu_mu);
    set_device();
    quiesce();
    L.export_lists(nlist, list_off, store, out_codes, out_ids);
  }
  void pack_lists(int64_t* list_off, void* out_ids, uint8_t* out_rows) override {
    RwSharedGuard rl(this);
    std::lock_guard<std::mutex> gl(gpu_mu);
    set_device();
    quiesce();
    L.pack(nlist, list_off, store, out_ids, out_rows);
  }
};

IndexBase* make_ivf_pq(b200vs_metric m, int d, const b200vs_params& p) { return new IvfPqIndex(m, d, p); }

static IvfPqIndex* as_ivf_pq(IndexBase* ix) {
  auto* p = dynamic_cast<IvfPqIndex*>(ix);
  if (!p) fail(B200VS_EINTERNAL, "not an IVF_PQ index");
  return p;
}

int ivf_pq_ksub(IndexBase* ix) { return as_ivf_pq(ix)->ksub; }

void ivf_pq_train_coarse(IndexBase* ix, int64_t n, const float* x, int k, std::vector<float>& cent) {
  IvfPqIndex* p = as_ivf_pq(ix);
  WriteHold hold(p);
  p->train_coarse_locked(n, x, k, cent);
}

void ivf_pq_train_state(IndexBase* ix, int64_t n, const float* x, const std::vector<float>& cent, std::vector<unsigned char>& blob) {
  IvfPqIndex* p = as_ivf_pq(ix);
  std::vector<float> cb;
  {
    WriteHold hold(p);
    p->train_codebooks_locked(n, x, cent, cb);
  }
  const int64_t hdr[6] = {0x51505649, (int64_t)(cent.size() / p->dim), p->dim, (int64_t)p->metric, p->M, p->nbits};
  blob.resize(48 + (cent.size() + cb.size()) * 4);
  memcpy(blob.data(), hdr, 48);
  memcpy(blob.data() + 48, cent.data(), cent.size() * 4);
  memcpy(blob.data() + 48 + cent.size() * 4, cb.data(), cb.size() * 4);
}

}  // namespace b200vs
