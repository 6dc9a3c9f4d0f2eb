// rebuild.cu — the device pieces of b200vs_rebuild_from shared by every index type: the live rows of an index in ascending
// id order, the training subsample drawn from device rows, and the +-1 expansion of binary rows.
#include <cub/cub.cuh>

#include "index.h"
#include "ivf_common.h"

namespace b200vs {

namespace {

__global__ void gather_words_kernel(const uint32_t* __restrict__ src, const long long* __restrict__ rows, long long n, int words,
                                    uint32_t* __restrict__ dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * words) return;
  const long long r = i / words;
  const int j = (int)(i % words);
  const long long sr = rows ? rows[r] : r;
  dst[i] = src[(size_t)sr * words + j];
}

// bit b of a padded row is bit (b & 31) of word b >> 5 (byte b >> 3 is byte (b >> 3) & 3 of that little-endian word)
__global__ void expand_pm1_kernel(const uint32_t* __restrict__ words, const long long* __restrict__ rows, long long m, int w, int dim,
                                  float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m * dim) return;
  const long long r = i / dim;
  const int b = (int)(i % dim);
  const long long sr = rows ? rows[r] : r;
  out[i] = ((words[(size_t)sr * w + (b >> 5)] >> (b & 31)) & 1u) ? 1.0f : -1.0f;
}

}  // namespace

void launch_gather_words(const uint32_t* src, const long long* rows, int64_t n, int words, uint32_t* dst, cudaStream_t s) {
  if (n <= 0) return;
  gather_words_kernel<<<(unsigned)cdiv(n * words, 256), 256, 0, s>>>(src, rows, n, words, dst);
  B200VS_CUDA(cudaGetLastError());
}

void launch_expand_pm1(const uint32_t* words, const long long* rows, int64_t m, int w, int dim, float* out, cudaStream_t s) {
  if (m <= 0) return;
  expand_pm1_kernel<<<(unsigned)cdiv(m * dim, 256), 256, 0, s>>>(words, rows, m, w, dim, out);
  B200VS_CUDA(cudaGetLastError());
}

int64_t kmeans_sample_rows(IndexBase* ix, int64_t n, int k, int max_pts, int64_t seed, DevBuf<long long>& out) {
  if (n <= (int64_t)k * max_pts) return n;
  std::vector<int64_t> perm;
  kmeans_rand_perm(perm, n, seed);
  const int64_t m = (int64_t)k * max_pts;
  out.reserve(m, 0, ix->stream);
  B200VS_CUDA(cudaMemcpyAsync(out.p, perm.data(), (size_t)m * 8, cudaMemcpyHostToDevice, ix->stream));
  B200VS_CUDA(cudaStreamSynchronize(ix->stream));  // perm dies here
  return m;
}

void sorted_live_rows(IndexBase* ix, int64_t n, const long long* ids, const long long* slots, bool on_device, const uint32_t* src,
                      int words, DevBuf<uint32_t>& out_rows, DevBuf<long long>& out_ids, cudaStream_t s) {
  if (n == 0) return;
  if (n >= (1LL << 31)) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild holds at most 2^31 - 1 rows");
  DevBuf<long long> keys, vals, sorted_slots;
  const long long* k_in = ids;
  const long long* v_in = slots;
  if (!on_device) {
    keys.reserve(n, 0, s); vals.reserve(n, 0, s);
    B200VS_CUDA(cudaMemcpyAsync(keys.p, ids, (size_t)n * 8, cudaMemcpyHostToDevice, s));
    B200VS_CUDA(cudaMemcpyAsync(vals.p, slots, (size_t)n * 8, cudaMemcpyHostToDevice, s));
    k_in = keys.p; v_in = vals.p;
  } else if (!slots) {  // the rows' own positions
    vals.reserve(n, 0, s);
    launch_iota(vals.p, n, s);
    v_in = vals.p;
  }
  sorted_slots.reserve(n, 0, s); out_ids.reserve(n, 0, s);
  size_t tmp_bytes = 0;
  B200VS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, k_in, out_ids.p, v_in, sorted_slots.p, (int)n, 0, 64, s));
  DevBuf<unsigned char> tmp;
  tmp.reserve(std::max<size_t>(tmp_bytes, 1), 0, s);
  B200VS_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, k_in, out_ids.p, v_in, sorted_slots.p, (int)n, 0, 64, s));
  out_rows.reserve((size_t)n * words, 0, s);
  launch_gather_words(src, sorted_slots.p, n, words, out_rows.p, s);
  B200VS_CUDA(cudaStreamSynchronize(s));  // the host id and slot lists and the sort's buffers die here
  ix->launch_count(3);
}

void check_rebuild_pair(const IndexBase& dst, const IndexBase& src) {
  if (&dst == &src) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from: dst and src are the same index");
  if (dst.type != src.type || dst.metric != src.metric || dst.dim != src.dim)
    fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from: dst and src differ in type, metric or dimension");
  // the creation parameters that decide this type's results, resolved (<= 0 = the default): an index created with the
  // default and one created with the default's value are the same index
  const b200vs_params &a = dst.params, &b = src.params;
  auto same = [](int64_t x, int64_t y, int64_t dflt) { return (x > 0 ? x : dflt) == (y > 0 ? y : dflt); };
  const bool ivf = dst.type == B200VS_IVF_FLAT || dst.type == B200VS_BINARY_IVF_FLAT || dst.type == B200VS_IVF_PQ;
  bool ok = dst.device == src.device;
  if (ivf) ok = ok && same(a.nlist, b.nlist, 2048);
  if (dst.type == B200VS_IVF_PQ) ok = ok && same(a.pq_m, b.pq_m, 64) && same(a.pq_nbits, b.pq_nbits, 8);
  if (dst.type == B200VS_HNSW) ok = ok && a.hnsw_m == b.hnsw_m && a.hnsw_efc == b.hnsw_efc;
  if (!ok) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from: dst and src differ in nlist, nsubvector, nbits, nlinks, efconstruction or device");
  if ((ivf && dst.is_trained()) || dst.count() != 0 || dst.deleted_count() != 0)
    fail(B200VS_EILLEGAL_PARAMETERS, "rebuild_from: dst must be empty and untrained");
}

}  // namespace b200vs
