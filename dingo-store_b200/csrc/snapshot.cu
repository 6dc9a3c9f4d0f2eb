// snapshot.cu — the parent's half of a fork-based snapshot (b200vs_save_stage): the bytes b200vs_save would write, built in
// pageable host memory with one device pack of the live rows.  The child's half, the file write, is snapshot_write.cc.
#include <algorithm>

#include "index.h"
#include "ivf_common.h"

namespace b200vs {

namespace {

// One warp per output row: row r is the first epr elements of source row slots[r], and its id comes along.  T is the widest
// word that divides both the source pitch and the output row, so FP32 rows, PQ code rows and the leading dim / 8 bytes of a
// padded binary row all move as wide, coalesced loads.
template <class T>
__global__ void pack_rows_kernel(const unsigned char* __restrict__ src, size_t pitch, const long long* __restrict__ src_ids,
                                 const long long* __restrict__ slots, int64_t n, int epr, T* __restrict__ out,
                                 long long* __restrict__ out_ids) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += warps) {
    const long long s = slots[r];
    const T* in = reinterpret_cast<const T*>(src + (size_t)s * pitch);
    T* o = out + (size_t)r * epr;
    for (int e = lane; e < epr; e += 32) o[e] = in[e];
    if (lane == 0) out_ids[r] = src_ids[s];
  }
}

template <class T>
void launch_pack(const void* src, size_t pitch, const long long* src_ids, const long long* slots, int64_t n, size_t row_bytes, void* out,
                 long long* out_ids, cudaStream_t s) {
  const int64_t blocks = std::min<int64_t>(cdiv(n, 8), 132 * 32);
  pack_rows_kernel<T><<<(unsigned)blocks, 256, 0, s>>>(static_cast<const unsigned char*>(src), pitch, src_ids, slots, n,
                                                       (int)(row_bytes / sizeof(T)), static_cast<T*>(out), out_ids);
  B200VS_CUDA(cudaGetLastError());
}

}  // namespace

void pack_rows(IndexBase* ix, const std::vector<long long>& slots, const void* rows, size_t pitch, const long long* ids, size_t row_bytes,
               void* out_ids, uint8_t* out_rows) {
  const int64_t n = (int64_t)slots.size();
  if (n == 0) return;
  cudaStream_t s = ix->stream;
  // rows are packed in chunks of at most 1 GiB, so a large index needs no second copy of its rows on the device; a region
  // (512 MB at the auto-split size) is one chunk
  const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(n, ((int64_t)1 << 30) / (int64_t)row_bytes));
  DevBuf<long long> d_slots, d_ids;
  DevBuf<unsigned char> d_rows;
  d_slots.reserve(n, 0, s);
  d_ids.reserve(n, 0, s);
  d_rows.reserve((size_t)chunk * row_bytes, 0, s);
  B200VS_CUDA(cudaMemcpyAsync(d_slots.p, slots.data(), (size_t)n * 8, cudaMemcpyHostToDevice, s));
  const size_t both = pitch | row_bytes;  // its low bits are zero where both sizes' are: the widest word dividing both
  for (int64_t a = 0; a < n; a += chunk) {
    const int64_t m = std::min(chunk, n - a);
    if (both % 16 == 0) launch_pack<uint4>(rows, pitch, ids, d_slots.p + a, m, row_bytes, d_rows.p, d_ids.p + a, s);
    else if (both % 8 == 0) launch_pack<uint2>(rows, pitch, ids, d_slots.p + a, m, row_bytes, d_rows.p, d_ids.p + a, s);
    else if (both % 4 == 0) launch_pack<uint32_t>(rows, pitch, ids, d_slots.p + a, m, row_bytes, d_rows.p, d_ids.p + a, s);
    else launch_pack<uint8_t>(rows, pitch, ids, d_slots.p + a, m, row_bytes, d_rows.p, d_ids.p + a, s);
    ix->launch_count(1);
    B200VS_CUDA(cudaMemcpyAsync(out_rows + (size_t)a * row_bytes, d_rows.p, (size_t)m * row_bytes, cudaMemcpyDeviceToHost, s));
  }
  B200VS_CUDA(cudaMemcpyAsync(out_ids, d_ids.p, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
  B200VS_CUDA(cudaStreamSynchronize(s));
}

// IndexBase::save's container, byte for byte: header, trained-state blob, list offsets, ids, rows
void IndexBase::save_image(SnapshotImage& img) {
  RwSharedGuard hold(this);  // one reader hold across count / trained state / pack, as in save
  const int64_t st_len = std::max<int64_t>(get_state(nullptr, 0), 0);
  const int nl = export_nlist();
  const int64_t n = type == B200VS_HNSW ? 0 : count();  // the HNSW blob already carries rows + labels
  const size_t rb = query_row_bytes();
  IndexFileHdr h;
  memcpy(h.magic, binary() ? "B2VSBIN1" : "B2VSIDX1", 8);
  h.type = type; h.metric = metric; h.dim = dim; h.nlist = nl; h.state_len = st_len; h.count = n;
  const size_t off_at = sizeof(h) + (size_t)st_len, ids_at = off_at + ((size_t)nl + 1) * 8, rows_at = ids_at + (size_t)n * 8;
  img.alloc(rows_at + (size_t)n * rb);
  uint8_t* p = img.bytes.get();
  memcpy(p, &h, sizeof(h));
  if (st_len > 0) get_state(p + sizeof(h), (size_t)st_len);
  std::vector<int64_t> off((size_t)nl + 1, 0);
  if (n) pack_lists(off.data(), p + ids_at, p + rows_at);
  memcpy(p + off_at, off.data(), off.size() * 8);
}

}  // namespace b200vs
