// deep_select.cuh — the key sink of the exact scans for deep top-k (k above what a shared-memory select holds).
//
// A deep search runs the exact scan kernels (scan_rows in scan_kernels.cuh, the IVF-PQ LUT scans) with this sink in place
// of SelectSink: every eligible candidate's 32-bit key (f2ord of the L2 / Hamming distance, or of -ip) is written at its
// position in the query's candidate space, and its eligibility beside it.  The select passes of deep_select.cu then run
// over those keys in global memory.  The per-row arithmetic is the select path's own, so the keys are equal by construction.
#pragma once
#include "common.cuh"

namespace b200vs {

// The key buffers of one query chunk.  A query's candidate space is its row index [0, n) on a dense scan, or its
// probe-prefix position (the rows of probe p follow those of probes 0 .. p-1, in list order) on a list scan.
struct DeepKeys {
  uint32_t* keys;              // [nqc, stride]
  unsigned char* elig;         // [nqc, stride], 1 = the candidate is a live row that passes the filters (zeroed before)
  unsigned long long* count;   // [nqc] eligible candidates (zeroed before)
  long long stride;            // the largest candidate space of the chunk
  const long long* pre;        // list scans: [nqc, nprobe + 1] probe-prefix positions; null on a dense scan
  int nprobe;
};

struct DeepKeySink {
  uint32_t* keys;
  unsigned char* elig;
  unsigned long long* count;
  const long long* pre;
  unsigned n = 0;
  __device__ DeepKeySink(const DeepKeys& o, int q)
      : keys(o.keys + (size_t)q * o.stride), elig(o.elig + (size_t)q * o.stride), count(o.count + q),
        pre(o.pre ? o.pre + (size_t)q * (o.nprobe + 1) : nullptr) {}
  __device__ void init(unsigned char*) { __syncthreads(); }
  // the candidate-space position of row 0 of probe p (list scans)
  __device__ __forceinline__ long long list_pos(int p) const { return pre[p]; }
  __device__ __forceinline__ void step(int) {}
  __device__ __forceinline__ void take(uint32_t key, long long, long long pos) {
    keys[pos] = key;
    elig[pos] = 1;
    ++n;
  }
  // all threads of the block call, converged
  __device__ void finish() {
    unsigned v = n;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(count, (unsigned long long)v);
  }
};

}  // namespace b200vs
