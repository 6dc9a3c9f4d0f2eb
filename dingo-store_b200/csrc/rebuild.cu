// rebuild.cu — the device pieces of b200vs_rebuild_from[_range] shared by every index type: the live rows of one or more
// indexes in an id range in ascending id order, the training subsample drawn from device rows, and the +-1 expansion of
// binary rows.
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

// a rebuild's sort value: the source in the top bits, the row slot in its store below
constexpr int kSlotBits = 56;
constexpr long long kSlotMask = (1LL << kSlotBits) - 1;
static_assert(kRebuildMaxSources <= (1 << (63 - kSlotBits)), "the source must fit above the slot");

struct SourceRows {
  const uint32_t* p[kRebuildMaxSources];  // each source's row store
};

// out row r = row (vals[r] & kSlotMask) of source vals[r] >> kSlotBits, one warp per row in T-sized pieces (wt per row).
// dup (nullable) is set when rows r - 1 and r share an id but come from different sources: the sort keeps equal ids of one
// source together behind each other, so an id held by two sources always meets such a pair.
template <class T>
__global__ void gather_sources_kernel(const __grid_constant__ SourceRows src, const long long* __restrict__ vals,
                                      const long long* __restrict__ ids, long long n, int wt, T* __restrict__ out, int* __restrict__ dup) {
  const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const long long v = vals[r];
  const T* row = reinterpret_cast<const T*>(src.p[v >> kSlotBits]) + (size_t)(v & kSlotMask) * wt;
  T* o = out + (size_t)r * wt;
  for (int j = lane; j < wt; j += 32) o[j] = row[j];
  if (dup && lane == 0 && r > 0 && ids[r] == ids[r - 1] && (vals[r - 1] >> kSlotBits) != (v >> kSlotBits)) *dup = 1;
}

// the stable sort of n (id, source | slot) pairs by id and the gather of their rows; refuses an id held by two sources
void sort_gather(IndexBase* ix, int64_t n, const long long* keys, const long long* vals, const SourceRows& src, int nsrc, int words,
                 DevBuf<uint32_t>& out_rows, DevBuf<long long>& out_ids, cudaStream_t s) {
  DevBuf<long long> sorted_vals;
  sorted_vals.reserve(n, 0, s); out_ids.reserve(n, 0, s);
  DevBuf<unsigned char> tmp;
  sort_by_id(n, keys, out_ids.p, vals, sorted_vals.p, [&](size_t bytes) -> void* { tmp.reserve(std::max<size_t>(bytes, 1), 0, s); return tmp.p; }, s);
  out_rows.reserve((size_t)n * words, 0, s);
  DevBuf<int> dup;
  if (nsrc > 1) {
    dup.reserve(1, 0, s);
    B200VS_CUDA(cudaMemsetAsync(dup.p, 0, 4, s));
  }
  const unsigned blocks = (unsigned)cdiv(n, 8);  // 8 warps of 256 threads, a row each
  if (words % 4 == 0)  // 16-byte rows: every row of a cudaMalloc'ed store starts 16-byte aligned
    gather_sources_kernel<uint4><<<blocks, 256, 0, s>>>(src, sorted_vals.p, out_ids.p, n, words / 4, reinterpret_cast<uint4*>(out_rows.p), dup.p);
  else
    gather_sources_kernel<uint32_t><<<blocks, 256, 0, s>>>(src, sorted_vals.p, out_ids.p, n, words, out_rows.p, dup.p);
  B200VS_CUDA(cudaGetLastError());
  int h_dup = 0;
  if (dup.p) B200VS_CUDA(cudaMemcpyAsync(&h_dup, dup.p, 4, cudaMemcpyDeviceToHost, s));
  B200VS_CUDA(cudaStreamSynchronize(s));  // the key and value lists and the sort's buffers die here
  ix->launch_count(3);
  if (h_dup) fail(B200VS_EVECTOR_ID_DUPLICATED, "rebuild_from_range: an id in the range is held by more than one source");
}

// out[i] = tag | i: the sort values of one block of device rows (the block in the tag's top bits, as in sort_gather)
__global__ void source_slots_kernel(long long* __restrict__ out, long long n, long long tag) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = tag | i;
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

void sort_by_id(int64_t n, const long long* keys, long long* keys_out, const long long* vals, long long* vals_out,
                const std::function<void*(size_t)>& temp, cudaStream_t s) {
  if (n >= (1LL << 31)) fail(B200VS_EILLEGAL_PARAMETERS, "a sort by id holds at most 2^31 - 1 rows");
  size_t tmp_bytes = 0;
  B200VS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys, keys_out, vals, vals_out, (int)n, 0, 64, s));
  void* tmp = temp(tmp_bytes);
  B200VS_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, keys_out, vals, vals_out, (int)n, 0, 64, s));
}

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

int64_t sorted_live_rows(IndexBase* ix, const std::vector<IndexBase*>& srcs, int64_t lo, int64_t hi, int words, DevBuf<uint32_t>& out_rows,
                         DevBuf<long long>& out_ids, cudaStream_t s) {
  if (srcs.empty() || srcs.size() > (size_t)kRebuildMaxSources) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild takes 1 to 16 sources");
  std::vector<RebuildSource> parts(srcs.size());  // holds inner indexes' reader locks until the gather is done
  // in address order, as the callers take the outer locks: the inner locks some sources take here follow that one order too
  std::vector<size_t> order(srcs.size());
  for (size_t k = 0; k < srcs.size(); ++k) order[k] = k;
  std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return std::less<IndexBase*>()(srcs[a], srcs[b]); });
  int64_t n = 0;
  for (size_t k : order) {
    srcs[k]->live_rows(lo, hi, parts[k]);
    n += (int64_t)parts[k].ids.size();
  }
  if (n == 0) return 0;
  if (n >= (1LL << 31)) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild holds at most 2^31 - 1 rows");
  std::vector<long long> keys, vals;
  keys.reserve(n); vals.reserve(n);
  SourceRows table{};
  for (size_t k = 0; k < parts.size(); ++k) {
    const RebuildSource& p = parts[k];
    for (size_t i = 0; i < p.ids.size(); ++i) {
      if (p.slots[i] > kSlotMask) fail(B200VS_EINTERNAL, "rebuild: row slot out of range");
      keys.push_back(p.ids[i]);
      vals.push_back(((long long)k << kSlotBits) | p.slots[i]);
    }
    table.p[k] = p.rows;
    if (!p.ids.empty()) B200VS_CUDA(cudaStreamSynchronize(p.stream));  // every write the source's own stream holds
  }
  DevBuf<long long> d_keys, d_vals;
  d_keys.reserve(n, 0, s); d_vals.reserve(n, 0, s);
  B200VS_CUDA(cudaMemcpyAsync(d_keys.p, keys.data(), (size_t)n * 8, cudaMemcpyHostToDevice, s));
  B200VS_CUDA(cudaMemcpyAsync(d_vals.p, vals.data(), (size_t)n * 8, cudaMemcpyHostToDevice, s));
  sort_gather(ix, n, d_keys.p, d_vals.p, table, (int)srcs.size(), words, out_rows, out_ids, s);
  return n;
}

void sorted_live_rows(IndexBase* ix, const std::vector<DeviceRows>& blocks, int words, DevBuf<uint32_t>& out_rows, DevBuf<long long>& out_ids,
                      cudaStream_t s) {
  if (blocks.empty() || blocks.size() > (size_t)kRebuildMaxSources) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild takes 1 to 16 sources");
  int64_t n = 0;
  for (const DeviceRows& b : blocks) n += b.n;
  if (n == 0) return;
  if (n >= (1LL << 31)) fail(B200VS_EILLEGAL_PARAMETERS, "rebuild holds at most 2^31 - 1 rows");
  // keys: the blocks' ids back to back (one block: its own ids); values: (block, the row's position in its block)
  DevBuf<long long> keys, vals;
  vals.reserve(n, 0, s);
  if (blocks.size() > 1) keys.reserve(n, 0, s);
  SourceRows table{};
  int64_t at = 0;
  for (size_t k = 0; k < blocks.size(); ++k) {
    const DeviceRows& b = blocks[k];
    table.p[k] = b.rows;
    if (!b.n) continue;
    if (keys.p) B200VS_CUDA(cudaMemcpyAsync(keys.p + at, b.ids, (size_t)b.n * 8, cudaMemcpyDeviceToDevice, s));
    source_slots_kernel<<<(unsigned)cdiv(b.n, 256), 256, 0, s>>>(vals.p + at, b.n, (long long)k << kSlotBits);
    B200VS_CUDA(cudaGetLastError());
    at += b.n;
  }
  sort_gather(ix, n, keys.p ? keys.p : blocks[0].ids, vals.p, table, (int)blocks.size(), words, out_rows, out_ids, s);
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
