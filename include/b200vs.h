/*
 * b200vs.h — C ABI of the H100-native vector-search engine (libb200vs.so).
 *
 * This is the drop-in boundary behind dingo-store's C++ VectorIndex plugin surface
 * (reference: src/vector/vector_index.h:56-279).  A thin C++ subclass of dingodb::VectorIndex
 * (dingo-store_b200/host/vector_index_b200.{h,cc}; binding shown in INTEGRATION.md) marshals protobuf
 * to flat arrays and calls these entry points; everything below the ABI is CUDA for sm_90a.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes only.  No exception or abort crosses the ABI: every entry
 *     point returns a b200vs_status; b200vs_last_error() gives a thread-local message.
 *   - Status codes map 1:1 to the pb::error::Errno classes the reference plugins return
 *     (src/vector/vector_index_flat.cc:209, :193-196; vector_index_ivf_flat.cc:112; vector_index_hnsw.cc:332-336,
 *     :487-493; vector_index_utils.cc:551-561).
 *   - Unless a function name ends in _device, all data pointers are HOST pointers.
 *   - Distances are returned in the reference's API semantics (src/vector/vector_index_utils.cc:611-655):
 *     L2 = squared L2; INNER_PRODUCT and COSINE = 1 - ip.  Results are ascending; rows with fewer than k
 *     hits are padded with id = -1, dist = 0 (labels pre-filled -1, vector_index_flat.cc:218-219).
 *   - Thread-safety: searches may be issued concurrently from many host threads (the reference calls
 *     Search from a 16-thread pool, src/server/server.cc:868-873); writers are serialised against readers
 *     by a reader/writer lock inside the index (reference: RWLock, src/common/synchronization.h:133-156).
 */
#ifndef B200VS_H_
#define B200VS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200vs_index b200vs_index; /* opaque */

/* replaces VectorIndexFactory::New type switch, src/vector/vector_index_factory.cc:40-95 */
typedef enum {
  B200VS_FLAT = 0, B200VS_IVF_FLAT = 1, B200VS_IVF_PQ = 2, B200VS_HNSW = 3,
  /* VECTOR_INDEX_TYPE_BINARY_FLAT / _BINARY_IVF_FLAT (vector_index_factory.cc:73-80): faiss IndexBinaryFlat under
   * IndexBinaryIDMap2 and IndexBinaryIVF.  dim counts BITS (dim % 8 == 0, 0 < dim <= 32768); rows are packed, dim / 8 bytes
   * each, byte j = binary_values[j] (vector_index_utils.cc:597-599); metric must be B200VS_HAMMING.  They are served by the
   * b200vs_*_binary entry points; the float ones refuse them (EILLEGAL_PARAMETERS), and vice versa. */
  B200VS_BINARY_FLAT = 4, B200VS_BINARY_IVF_FLAT = 5
} b200vs_type;
/* mirrors pb::common::MetricType L2 / INNER_PRODUCT / COSINE / HAMMING */
typedef enum { B200VS_L2 = 1, B200VS_IP = 2, B200VS_COSINE = 3, B200VS_HAMMING = 4 } b200vs_metric;

typedef enum {
  B200VS_OK = 0,
  B200VS_EILLEGAL_PARAMETERS = 1, /* pb::error::EILLEGAL_PARAMTETERS */
  B200VS_EVECTOR_INVALID = 2,     /* pb::error::EVECTOR_INVALID       */
  B200VS_EVECTOR_NOT_TRAIN = 3,   /* pb::error::EVECTOR_NOT_TRAIN     */
  B200VS_EVECTOR_NOT_SUPPORT = 4, /* pb::error::EVECTOR_NOT_SUPPORT   */
  B200VS_EINTERNAL = 5,           /* pb::error::EINTERNAL             */
  B200VS_EVECTOR_ID_DUPLICATED = 6 /* pb::error::EVECTOR_ID_DUPLICATED */
} b200vs_status;

/* creation parameters: the union of pb::common::Create{Flat,IvfFlat,IvfPq,Hnsw}Param fields read at
 * vector_index_flat.cc:81-82, vector_index_ivf_flat.cc:75-83, vector_index_raw_ivf_pq.cc:60-75,
 * vector_index_hnsw.cc:141-182.  0 = reference default (src/common/constant.h:177-188). */
typedef struct {
  int32_t nlist;        /* ncentroids; default 2048 */
  int32_t pq_m;         /* nsubvector; default 64   */
  int32_t pq_nbits;     /* nbits_per_idx 1-8 (faiss bit-packed codes); <= 0 -> 8; 9-16 refused (EILLEGAL_PARAMETERS) */
  int32_t hnsw_m;       /* nlinks */
  int32_t hnsw_efc;     /* efconstruction */
  int64_t max_elements; /* hnsw max_elements */
  int32_t device;       /* CUDA device ordinal */
  int32_t hnsw_build_threads; /* host threads inserting a batch into the HNSW graph.  0 / 1 = single writer (deterministic
                               * graph, equal to the oracle's); > 1 = concurrent insertion with per-node locks, what the
                               * reference does with its 16-thread pool (vector_index_hnsw.cc:229-243: graph differs run to run) */
} b200vs_params;

/* search-time parameters: pb::common::VectorSearchParameter knobs (ivf_flat().nprobe() ivf_flat.cc:211,
 * ivf_pq().nprobe() raw_ivf_pq.cc:170, hnsw().efsearch() hnsw.cc:332) plus the device form of the
 * reference's FilterFunctors (vector_index.h:67-146): all given filters are ANDed. */
typedef struct {
  int32_t nprobe;   /* <=0 -> 80 (Constant::kSearchIvfFlatParamNprobe); clamped to nlist */
  int32_t efsearch; /* 0 -> keep the sticky ef; outside [0,1024] -> EILLEGAL_PARAMETERS */
  int32_t has_range; /* RangeFilterFunctor: range_min <= id < range_max */
  int32_t negate;    /* SortFilterFunctor / ConcreteFilterFunctor is_negation */
  int64_t range_min, range_max;
  const int64_t* sorted_ids; /* ascending id list (HOST pointer), or NULL */
  int64_t n_ids;
  int32_t exact_only; /* 1 = force the exact scan: FP32 on float indexes, Hamming on binary indexes (skip the tile scan) */
  int32_t reserved;
} b200vs_search_params;

/* lifecycle — replaces the plugin constructors / destructors */
int b200vs_create(b200vs_type type, b200vs_metric metric, int32_t dim, const b200vs_params* params, b200vs_index** out);
void b200vs_destroy(b200vs_index* idx);

/* VectorIndex::Train(std::vector<float>&) — vector_index_ivf_flat.cc:644-712, raw_ivf_pq.cc:457-500,
 * ivf_pq.cc:327-395.  x row-major [n,dim], RAW values (COSINE is normalised inside).  Flat/HNSW: no-op. */
int b200vs_train(b200vs_index* idx, int64_t n, const float* x);
/* Load / fetch trained state (IVF centroids, PQ codebooks, HNSW graph) as a flat blob — used to search the
 * SAME trained index as the CPU path.  Layouts: see DESIGN.md §Trained-state blobs. */
int b200vs_set_trained_state(b200vs_index* idx, const void* blob, size_t len);
int64_t b200vs_get_trained_state(b200vs_index* idx, void* blob, size_t cap); /* returns bytes needed/written, <0 on error */

/* VectorIndex::Add / Upsert / Delete — flat.cc:121-203, ivf_flat.cc:92-190, hnsw.cc:203-281.
 * ids must be unique within one call (EVECTOR_ID_DUPLICATED); upsert=1 removes pre-existing ids first.
 * Ids must be >= 0 on every index type and every add entry point (the device and sharded variants and b200vs_scan_push
 * too): a batch holding a negative id is refused with EILLEGAL_PARAMETERS ("vector id is negative: <id>") before anything
 * changes, since the scans read a negative id as a deleted row or an empty result slot. */
int b200vs_add_with_ids(b200vs_index* idx, int64_t n, const float* x, const int64_t* ids, int upsert);
int b200vs_remove_ids(b200vs_index* idx, int64_t n, const int64_t* ids, int64_t* n_removed);

/* HNSW Add / Upsert with the graph built on the GPU in deterministic batches (DESIGN.md §4.4).  Host pointers; same semantics
 * as b200vs_add_with_ids on an HNSW index: cosine rows are normalised, an id already present is replaced (its old node is
 * tombstoned), an id repeated within the call is not refused and its last row wins.  Rows go in in call order; every row of a
 * batch searches the graph as it was at the batch start and also links to the batch's earlier rows.  Batches hold
 * min(batch, rows already in the graph) rows, so they grow 1, 1, 2, 4, ... from an empty index.
 *   batch <= 0: the default, 2048 rows (measured at cfg4, DESIGN §4.4); larger values are capped at 8192.
 *   batch == 1: the graph b200vs_add_with_ids builds with one writer, byte for byte (data without exact distance ties).
 * Levels, entry point and max level always equal the host builder's.  Empty / null input and a non-HNSW index:
 * EILLEGAL_PARAMETERS; more rows than max_elements: EINTERNAL "exceeds max elements".  efconstruction, dimension and batch
 * must fit the kernels' 200 KB of shared memory (roughly efconstruction + batch <= 12800; efconstruction >= 1024 runs the
 * search's candidate-heap form), else EILLEGAL_PARAMETERS.  Every refusal leaves the index unchanged, and so does a call that
 * fails on the device (EINTERNAL, e.g. out of memory): the graph changes only once the whole call has run.  Takes the writer
 * lock. */
int b200vs_hnsw_add_batched(b200vs_index* idx, int64_t n, const float* x, const int64_t* ids, int32_t batch);
/* Diagnostics (tests only): cap the device scratch one b200vs_hnsw_add_batched call of this index may allocate beyond the graph
 * (bytes; 0 = no cap, the default).  A call that needs more fails with EINTERNAL, as on a device out of memory, at the
 * allocation that crosses the cap (the peer matrix grows with the batches, so this can be mid-call, after earlier batches ran),
 * and leaves the index as it was.  Non-HNSW index or bytes < 0: EILLEGAL_PARAMETERS. */
int b200vs_debug_hnsw_build_scratch_limit(b200vs_index* idx, int64_t bytes);

/* VectorIndex::Search — flat.cc:205-264, ivf_flat.cc:191-275, raw_ivf_pq.cc:157-210, hnsw.cc:318-485.
 * xq row-major [nq,dim] RAW; out_dist [nq,k], out_ids [nq,k]. */
int b200vs_search(b200vs_index* idx, int64_t nq, const float* xq, int32_t k, const b200vs_search_params* sp,
                  float* out_dist, int64_t* out_ids);
/* b200vs_search and b200vs_search_binary coalesce concurrent callers (SURVEY 8b): the unchanged reference slices every batch
 * into one-query tasks on its 16-thread pool (src/vector/vector_index.cc:54, :244-271), so the plugin sees many concurrent
 * nq = 1 calls.  Calls of <= 64 queries without id-list filters (and with profiling off) queue inside the library; the caller
 * that finds no leader active runs every compatible pending request (same k / nprobe / efsearch / exact_only / id range) as
 * ONE batch and hands the results back.
 * on: 1 / 0 switch it, < 0 only reads; stats (nullable): [0] batches run, [1] requests served through them. */
int b200vs_set_coalescing(b200vs_index* idx, int on, int64_t stats[2]);

/* Same, with xq / out_dist / out_ids DEVICE pointers on the index's device; enqueued on `stream`
 * (a cudaStream_t) and NOT synchronised when it returns.  stream == NULL runs the search on a library-owned stream and
 * returns only when the results are complete (it does not touch the legacy default stream).  The same holds for
 * b200vs_coarse_device and b200vs_search_probes_device. */
int b200vs_search_device(b200vs_index* idx, int64_t nq, const float* xq_dev, int32_t k,
                         const b200vs_search_params* sp, float* out_dist_dev, int64_t* out_ids_dev, void* stream);

/* Deep top-k: exact search for any k in [1, B200VS_DEEP_MAX_K], past the shared-memory select that bounds b200vs_search
 * (VectorReader::SearchVector over-fetches top_n x 10 rows for its scalar post-filter, vector_reader.cc:119-215, and the
 * service allows top_n * batch <= 40960, index_service.cc:197-211).  Host pointers, the arguments of b200vs_search /
 * b200vs_search_binary, and their results bit for bit wherever those answer: API distances (squared L2, 1 - ip, Hamming),
 * (distance, id) order with ties to the smaller id, -1 / 0 padding past the eligible rows, the same cosine normalisation and
 * the same probes from the index's coarse step.  Every search parameter applies (nprobe, id range, sorted id list, negate);
 * exact_only is accepted, the deep path is always exact.  Types: FLAT, IVF_FLAT, IVF_PQ (inner Flat and IVF-PQ modes),
 * BINARY_FLAT, BINARY_IVF_FLAT.  k <= 0: OK, nothing done; k > B200VS_DEEP_MAX_K or the wrong row type: EILLEGAL_PARAMETERS;
 * HNSW: EVECTOR_NOT_SUPPORT.  Never coalesced; runs as an ordinary reader.  Cost: one exact-scan pass per query chunk that
 * writes a 4-byte key per candidate, then radix-select passes over those keys (DESIGN.md 4.10).
 * b200vs_last_search_stats[0] counts the launches of the call, [1] is 0. */
#define B200VS_DEEP_MAX_K 40960
int b200vs_search_deep(b200vs_index* idx, int64_t nq, const float* xq, int32_t k, const b200vs_search_params* sp,
                       float* out_dist, int64_t* out_ids);
int b200vs_search_binary_deep(b200vs_index* idx, int64_t nq, const uint8_t* xq, int32_t k, const b200vs_search_params* sp,
                              float* out_dist, int64_t* out_ids);

/* VectorIndex::RangeSearch — flat.cc:267-323, ivf_flat.cc:278-368 (HNSW: EVECTOR_NOT_SUPPORT, hnsw.cc:487-493).
 * radius in API semantics (mapped 1-r for IP/COSINE, flat.cc:282-285).  At most max_results hits per
 * query are kept (closest first); out_counts[nq] receives the per-query hit count.  Flat / IVF-Flat batches of >= 16
 * queries run on the tile scan's range mode; the results (ids, distances, counts) are those of exact_only.  A NaN radius
 * (either sign) admits no row: every count 0, ids -1, distances 0, and nothing is launched. */
int b200vs_range_search(b200vs_index* idx, int64_t nq, const float* xq, float radius, int32_t max_results,
                        const b200vs_search_params* sp, float* out_dist, int64_t* out_ids, int32_t* out_counts);

/* Binary indexes (B200VS_BINARY_FLAT / B200VS_BINARY_IVF_FLAT): the same calls on packed rows x / xq [n, dim / 8].
 * Distances are the faiss int32 Hamming distances, returned as float (exact) and emitted as is, with no 1 - x
 * (FillSearchResult, vector_index_utils.cc:640-650).  Results are ordered by (distance, id).  train: Flat no-op; IVF trains
 * faiss IndexBinaryIVF-style (binary_to_real, L2 k-means on the +-1 rows, real_to_binary; nlist degenerates to 1 with fewer
 * rows than nlist).  range_search: radius is truncated toward zero and hits have distance < (int)radius
 * (IndexBinary::range_search, flat.cc:304-308).  Search of an untrained IVF index returns empty results. */
int b200vs_train_binary(b200vs_index* idx, int64_t n, const uint8_t* x);
int b200vs_add_with_ids_binary(b200vs_index* idx, int64_t n, const uint8_t* x, const int64_t* ids, int upsert);
int b200vs_search_binary(b200vs_index* idx, int64_t nq, const uint8_t* xq, int32_t k, const b200vs_search_params* sp,
                         float* out_dist, int64_t* out_ids);
int b200vs_search_binary_device(b200vs_index* idx, int64_t nq, const uint8_t* xq_dev, int32_t k, const b200vs_search_params* sp,
                                float* out_dist_dev, int64_t* out_ids_dev, void* stream);
int b200vs_range_search_binary(b200vs_index* idx, int64_t nq, const uint8_t* xq, float radius, int32_t max_results,
                               const b200vs_search_params* sp, float* out_dist, int64_t* out_ids, int32_t* out_counts);

/* Stored vectors by id — what VectorIndexHnsw::Search returns per hit when reconstruct = true (hnswlib getDataByLabel,
 * vector_index_hnsw.cc:383-395; cosine indexes never reconstruct, :469-472).  out [n, dim]; found[n] = 1 / 0 (unknown or
 * deleted id: row left untouched).  Implemented for HNSW and FLAT. */
int b200vs_reconstruct(b200vs_index* idx, int64_t n, const int64_t* ids, float* out, uint8_t* found);

/* VectorIndex::VectorIndexSubType (vector_index.h:238; vector_index_ivf_pq.cc:474): for IVF_PQ the index type actually
 * serving searches — B200VS_FLAT while the inner Flat index is in use, B200VS_IVF_PQ once trained on enough data; -1 =
 * untrained.  Other types return their own type. */
int b200vs_sub_type(b200vs_index* idx);

/* GetCount / GetDeletedCount / GetMemorySize / IsTrained / NeedTrain — vector_index.h:150-152,:199-200 */
int b200vs_count(b200vs_index* idx, int64_t* count);
int b200vs_deleted_count(b200vs_index* idx, int64_t* count);
int b200vs_memory_size(b200vs_index* idx, int64_t* bytes);
int b200vs_is_trained(b200vs_index* idx);
int32_t b200vs_dimension(b200vs_index* idx);

/* Save / Load — vector_index.h:168-170 (own container format, see DESIGN.md; faiss/hnswlib file
 * compatibility is SURVEY §8(f)-4, not built). */
int b200vs_save(b200vs_index* idx, const char* path);
int b200vs_load(b200vs_index* idx, const char* path);

/* Fork-based snapshots (VectorIndexSnapshotManager::SaveVectorIndexSnapshot: LockWrite, fork, Save in the child,
 * UnlockWrite in the parent).  A forked child cannot use the parent's CUDA context, so the save is split at the fork:
 *   save_stage   : in the parent, builds in ordinary pageable host memory the exact bytes b200vs_save would write now and
 *                  keeps them in the handle, replacing an earlier image.  The live rows are packed on the device and brought
 *                  back with one copy per buffer on the index's stream; HNSW needs no device work.  Runs under the index's
 *                  reader lock, as b200vs_save does.  A failed host allocation or device step returns EINTERNAL and leaves
 *                  no image (an earlier one is freed too).
 *   save_staged  : writes the staged image to path.  Safe in the forked child of a multi-threaded CUDA process: it calls
 *                  no CUDA function, takes no library lock (another parent thread may have held one at the fork), logs
 *                  nothing and starts no thread.  The file is byte-identical to what b200vs_save would have written at the
 *                  moment of save_stage; writes to the index after the stage do not change it, and b200vs_load reads it.
 *                  No image, or a null or empty path: EILLEGAL_PARAMETERS.  An I/O failure: EINTERNAL, the image is kept.
 *   save_unstage : frees the image; a no-op without one.  b200vs_destroy frees it too.
 * The caller serialises stage, staged write and unstage on one handle (the plugin does so under its write gate).  The image
 * costs one copy of the index's saved bytes in host memory while it is held. */
int b200vs_save_stage(b200vs_index* idx);
int b200vs_save_staged(b200vs_index* idx, const char* path);
void b200vs_save_unstage(b200vs_index* idx);

/* VectorIndex::NeedToRebuild (vector_index.h:198): 1 = rebuild, 0 = not, < 0 = a status negated.  The reference plugins' rules
 * (max_points_per_centroid = 256; count = live rows; train_rows = n of the b200vs_train[_binary] call that trained the index,
 * or the live count after b200vs_load or at b200vs_set_trained_state; it is not saved):
 *   IVF_FLAT, BINARY_IVF_FLAT (vector_index_ivf_flat.cc:751-776), nlist_org = the created nlist (default 2048):
 *                    untrained, or nlist == nlist_org == 1: 0; nlist degenerated to 1: count >= 256 * nlist_org;
 *                    nlist == nlist_org: count >= 256 * nlist_org and train_rows <= count / 2
 *   IVF_PQ           inner-Flat mode: count >= max(256 * nlist, 256 * 2^nbits) (b200vs_train's threshold for IVF-PQ);
 *                    IVF-PQ mode: count / 2 >= train_rows; untrained: 0 (ivf_pq.cc:411-436, raw_ivf_pq.cc:518-526)
 *   HNSW             deleted > 0 and deleted > (count + deleted) / 2 (vector_index_hnsw.cc:577-590)
 *   FLAT, BINARY_FLAT: 0 (vector_index_flat.h:111) */
int b200vs_need_rebuild(b200vs_index* idx);

/* Fill dst, a fresh index, from src's live rows on the device, in place of the host scan + b200vs_train + b200vs_add_with_ids
 * loop of VectorIndexManager::RebuildVectorIndex (vector_index_manager.cc:864-1013).  dst ends up equal, byte for byte, to a
 * fresh index trained and then filled with src's live rows in ascending id order (rows sharing an id in an IVF index keep
 * their list-major export order), the rows taken as stored: cosine rows are already normalised and are not normalised again.
 *   IVF_FLAT, BINARY_IVF_FLAT : b200vs_train[_binary]'s rule on those rows (nlist degenerates to 1 below nlist rows), then one
 *                               add of them
 *   IVF_PQ in inner-Flat mode : b200vs_train's rule (IVF-PQ from max(256 * nlist, 256 * 2^nbits) rows, else inner Flat), then
 *                               one add; IVF_PQ in IVF-PQ mode keeps only codes: EVECTOR_NOT_SUPPORT
 *   HNSW                      : b200vs_hnsw_add_batched with the default batch; levels from dst's fresh generator, no tombstones
 *   FLAT, BINARY_FLAT         : EVECTOR_NOT_SUPPORT
 * EILLEGAL_PARAMETERS: dst == src, dst not empty or (IVF types) already trained, a different type, metric, dimension, nlist,
 * nsubvector, nbits, nlinks, efconstruction or device, or an HNSW dst whose max_elements is below src's live rows.  Every
 * refusal leaves both indexes unchanged.  An empty src: OK, dst stays untrained.  A device failure: EINTERNAL; dst may then be
 * discarded, src is unchanged.  src is held under its reader lock (its searches go on, its writers wait), dst under its
 * writer lock (the inner Flat index of an IVF_PQ src under its own reader lock too).  *n_rows (nullable) = rows copied.
 * Peak device memory: src's rows, a dense copy of its live rows (n x row bytes) with 32 B per row of sort buffers, and dst's
 * rows, all at once: about three times the live row bytes for IVF_FLAT (plus each IVF-Flat store's FP16 mirror).  A region
 * that does not fit that on its device (e.g. 6.25 M x 1536 FP32 = 38 GB of rows on an 80 GB GPU) keeps the host rebuild;
 * the call then fails with EINTERNAL and leaves src unchanged.  This is b200vs_rebuild_from_range's code with one source and
 * every id (a row whose id is INT64_MAX included). */
int b200vs_rebuild_from(b200vs_index* dst, b200vs_index* src, int64_t* n_rows);

/* Fill dst, a fresh index, from the live rows with id_min <= id < id_max of the indexes srcs[0 .. n_src), on the device: the
 * rebuilds of a region split or merge (raft_apply_handler.cc:626-660, :1018-1035), whose rows are already held by the old
 * indexes (a split child: the share index; a split parent: its own index; a merge target: its own index and the sibling).
 * R = the union over every source of its live rows with id_min <= id < id_max (RangeFilterFunctor's and
 * DecodeRangeToVectorId's convention: id_max is exclusive).  dst ends up equal, byte for byte (trained state, every list's
 * ids and rows, the FP16 mirror, PQ codes, the HNSW graph), to a fresh index trained by its type's rule and then filled with
 * one add of R in ascending id order (rows sharing an id inside one IVF source keep that source's list-major export order),
 * the rows taken as stored: cosine rows are not normalised again.
 *   IVF_FLAT, BINARY_IVF_FLAT : b200vs_train[_binary]'s rule on R (nlist degenerates to 1 below nlist rows), then one add
 *   IVF_PQ in inner-Flat mode : b200vs_train's rule (IVF-PQ from max(256 * nlist, 256 * 2^nbits) rows, else inner Flat), then
 *                               one add; a source in IVF-PQ mode keeps only codes: EVECTOR_NOT_SUPPORT
 *   HNSW                      : b200vs_hnsw_add_batched with the default batch; levels from dst's fresh generator, no tombstones
 *   FLAT, BINARY_FLAT         : one add (b200vs_rebuild_from keeps refusing them)
 * With one source and [0, INT64_MAX) the result equals b200vs_rebuild_from's on every type that call serves; only a row whose
 * id is INT64_MAX differs, and dingo never issues that id (IsLegalVectorId).
 * EILLEGAL_PARAMETERS: n_src outside [1, 16], a null srcs or null entry, id_min > id_max, dst among the sources, a source
 * listed twice, a source that differs from dst in type, metric, dimension, nlist, nsubvector, nbits, nlinks, efconstruction
 * or device, a dst that is not empty or (IVF types) already trained, or an HNSW dst whose max_elements is below |R|.
 * EVECTOR_ID_DUPLICATED: an id in R held by more than one source (the sources of a split or merge hold disjoint ranges).
 * Every refusal leaves every source and dst unchanged.  An empty R (id_min == id_max included): OK, *n_rows = 0, dst stays
 * untrained.  A device failure: EINTERNAL; the sources are unchanged, dst may be discarded.  The sources are held under their
 * reader locks (their searches go on, their writers wait) and dst under its writer lock, all taken in one order (by handle
 * address), so two calls over overlapping sources, such as a split's child and parent rebuilding from the same index at
 * once, cannot deadlock.  An IVF_PQ source in inner-Flat mode takes its writes under its inner index's lock only: that lock
 * is held shared (in the same address order) while the source's rows are listed and gathered, so its writers wait for that
 * part of the call, not for all of it.  *n_rows (nullable) = |R|.  Peak device memory: the sources' rows, a dense copy of R (|R| x row
 * bytes) with 32 B per row of sort buffers, and dst's rows, all at once: about three times R's row bytes for IVF_FLAT (plus
 * each IVF-Flat store's FP16 mirror) when the sources hold little beyond R. */
int b200vs_rebuild_from_range(b200vs_index* dst, int32_t n_src, b200vs_index* const* srcs, int64_t id_min, int64_t id_max,
                              int64_t* n_rows);

/* Export the inverted lists in list-major order (list l owns rows [list_off[l], list_off[l+1])) so a CPU
 * implementation can search the identical index.  Any output pointer may be NULL.  Flat: nlist = 1. */
int b200vs_export_lists(b200vs_index* idx, int64_t* list_off /*[nlist+1]*/, float* vectors /*[count,dim]*/,
                        uint8_t* codes /*[count, ceil(pq_m*pq_nbits/8)]; binary: [count, dim/8], vectors must be NULL*/,
                        int64_t* ids /*[count]*/);

/* One inverted list (live rows only, stored order): writes up to `cap` rows into vectors [cap, dim] / ids [cap] (either may
 * be NULL) and the list's live row count into *count.  Lets a checker rebuild exactly the lists a query probes without
 * copying a 77 GB shard to the host. */
int b200vs_export_list(b200vs_index* idx, int32_t list, int64_t cap, float* vectors, int64_t* ids, int64_t* count);

/* k-way merge of per-shard top-k, the engine's analogue of VectorIndexWrapper::MergeSearchResults
 * (src/vector/vector_index.cc:1056-1108).  parts_* are DEVICE arrays [nparts, nq, k] (API-semantics
 * distances ascending, id -1 padded) e.g. the output of one ncclAllGather; out_* DEVICE [nq,k]. */
int b200vs_merge_topk_device(int32_t device, int32_t nparts, int64_t nq, int32_t k, const float* parts_dist,
                             const int64_t* parts_ids, float* out_dist, int64_t* out_ids, void* stream);

/* List-sharded multi-GPU building blocks (IVF_FLAT, and IVF_PQ in its IVF-PQ mode; an IVF_PQ index in inner-Flat mode has
 * no lists and returns EVECTOR_NOT_SUPPORT): every rank holds all centroids but owns only some lists.
 * b200vs_coarse_device ranks the centroid rows [list_begin, list_end) only (this rank's share of the coarse work):
 * out_lists = GLOBAL list ids, out_score = the ranking score (L2 distance, or -ip: exact and ascending, so no
 * rounding can reorder ties), both [nq, nprobe] in (score, list id) order, so the per-rank
 * results can be all-gathered and merged with b200vs_merge_topk_device into the global top-nprobe
 * (= faiss quantizer->search(nq, x, nprobe), vector_index_ivf_flat.cc:247-251).  b200vs_search_probes_device then scans
 * the probed lists this rank owns for those (caller-supplied) probes (IVF_PQ: the coarse value each LUT scan starts from is
 * recomputed per (query, probe) with the coarse pass's arithmetic, so the results are b200vs_search's bit for bit). */
int b200vs_coarse_device(b200vs_index* idx, int64_t nq, const float* xq_dev, int32_t nprobe, int32_t list_begin, int32_t list_end,
                         float* out_score_dev, int64_t* out_lists_dev, void* stream);
int b200vs_search_probes_device(b200vs_index* idx, int64_t nq, const float* xq_dev, int32_t k, const int64_t* probes_dev, int32_t nprobe,
                                const b200vs_search_params* sp, float* out_dist_dev, int64_t* out_ids_dev, void* stream);

/* ---- List-sharded multi-GPU deployment (SURVEY.md 8e; one process per GPU) ----------------------------------------------
 * One LOGICAL IVF_FLAT or IVF_PQ index over `world` GPUs of one box: the trained state (centroids; IVF_PQ: and codebooks)
 * is replicated, rank r owns the inverted lists
 * [r * ceil(nlist / world), (r + 1) * ceil(nlist / world)) (b200vs_shard_list_range) — equivalently Raft regions mapped to
 * GPUs (src/vector/vector_index.h:54-55).  Every entry point below is COLLECTIVE: all ranks call it with the same
 * arguments (except the rows each rank contributes to add).  Communication is NCCL over NVLink, resolved at run time
 * (dlopen libnccl.so.2; override with B200VS_NCCL_LIB), one communicator per batch in flight.
 *   shard_unique_id : rank 0 creates the rendezvous blob; the host passes it to the other ranks out of band (dingo-store: RPC)
 *   shard_create    : wraps an (untrained or trained, still empty) IVF_FLAT or IVF_PQ index created with the GLOBAL nlist
 *                     (IVF_PQ in inner-Flat mode: EVECTOR_NOT_SUPPORT); `lanes` = batches that may be in flight (<= 0: 2);
 *                     world <= 1024 for every shard type (larger: EILLEGAL_PARAMETERS)
 *   shard_train     : distributed training — the row counts are exchanged first (fewer than nlist / world rows on any rank,
 *                     a null x counting as none, or for IVF_PQ fewer than 256 * 2^nbits on rank 0: EILLEGAL_PARAMETERS on
 *                     every rank, the index untouched); each rank clusters its rows into nlist / world centroids, one
 *                     all-gather.  IVF_PQ: rank 0 then trains the codebooks on its rows' residuals and its state is broadcast.
 *                     At world = 1 the state equals b200vs_train's.
 *   shard_broadcast_state : or: replicate rank `root`'s trained state (b200vs_train / b200vs_set_trained_state there); a root
 *                     without one: EVECTOR_NOT_TRAIN on every rank
 *   shard_add[_device]    : each rank passes the rows it holds; rows travel to the owner of their nearest centroid's list,
 *                     which receives rank 0's rows first, then rank 1's, ..., each in its caller's order
 *   shard_plan_add_device / shard_plan_commit : optional first pass of a bulk build (assignment only) that pre-sizes every
 *                     owned list in one allocation — a 77 GB shard cannot afford list relocation or arena re-allocation
 *   shard_search[_device] : all ranks pass the SAME batch.  Coarse quantiser on the rank's slice of the batch + all-gather of
 *                     the probe table; tile scan of the owned probed lists; ONE all-gather of the packed per-shard top-k
 *                     (16-byte (distance, id) records) + k-way merge (VectorIndexWrapper::MergeSearchResults,
 *                     src/vector/vector_index.cc:1056-1108): every rank returns the full merged [nq, k].  The host-pointer
 *                     variant uploads only the rank's slice of the batch and all-gathers the queries over NVLink.
 *                     seq = batch sequence number: 0, 1, 2, ... the same on every rank, each used exactly once: a refused
 *                     call, or one with k <= 0 (OK, nothing to do), still uses up its seq.  Batches are
 *                     enqueued in seq order on every rank (concurrent caller threads simply take turns; the GPU work of
 *                     up to `lanes` batches still overlaps), batch seq uses communicator seq % lanes.  seq < 0 = "next in
 *                     call order" for single-threaded callers.  Results equal b200vs_search on the unsharded index.
 *
 * Row-sharded FLAT and HNSW (DESIGN.md 4.5): the same entry points serve one logical FLAT or HNSW index.  A row belongs to
 * rank b200vs_row_owner(id) = splitmix64(id) mod world, so an upsert or a delete always meets the existing row on its owner,
 * and each rank's index keeps its type's single-index semantics.  On such a shard:
 *   shard_create    : accepts an EMPTY FLAT or HNSW index (a non-empty one: EVECTOR_NOT_SUPPORT)
 *   shard_train     : OK, nothing to do (as b200vs_train on FLAT and HNSW)
 *   shard_broadcast_state, shard_list_range, shard_plan_add_device, shard_plan_commit : EVECTOR_NOT_SUPPORT (no lists, and an
 *                     HNSW state is a whole graph)
 *   shard_add[_device] : every row travels raw to its owner, partitioned on the device; an owner receives rank 0's rows first,
 *                     then rank 1's, ..., each in its caller's order, and runs b200vs_add_with_ids on them in that order.
 *                     Before any index changes, every owner checks what it received (FLAT: an id repeated anywhere in the
 *                     collective call -> EVECTOR_ID_DUPLICATED; HNSW: more rows than max_elements -> EINTERNAL, and for
 *                     shard_hnsw_add_batched the batched builder's refusals for the rows received); every rank
 *                     then returns the same status and a refused call changes no rank's index
 *   shard_hnsw_add_batched : HNSW only; shard_add's routing, then b200vs_hnsw_add_batched(batch) on the received rows
 *   shard_remove_ids : unknown ids are ignored and the status is OK, as b200vs_remove_ids on FLAT and HNSW
 *   shard_search[_device] : no coarse step: the rank searches its own index with the whole batch (FLAT: b200vs_search's paths,
 *                     keyed on L2 distance | -ip, the API distance formed after the merge; HNSW: the graph walk with sp's
 *                     efsearch and filters, keyed on its own distance).  FLAT results equal b200vs_search on one index of all
 *                     rows bit for bit; HNSW results equal the merge of b200vs_search on every rank's graph.  Refused on
 *                     every rank before the first collective, from the arguments alone: HNSW efsearch outside [0, 1024]
 *                     (as b200vs_search) and a walk (max(efsearch or the index's current ef, k)) beyond the search
 *                     kernel's shared memory, also when this rank's graph is still empty; the refused efsearch is not kept.
 *   shard_range_search[_device] : FLAT: b200vs_range_search's rule, equal bit for bit.  HNSW: EVECTOR_NOT_SUPPORT on every
 *                     rank before the first collective (the sequence number is still used up).
 *
 * Snapshots of every shard kind (DESIGN.md 4.5).  Both calls are collectives of the write path: every rank passes the same
 * prefix (a path every rank can reach), they use up no search sequence number, and every rank returns the same status.
 *   shard_save : writes <prefix>.<r>-of-<W> per rank in b200vs_save's container (each one loads with plain b200vs_load) and
 *                <prefix>.manifest (rank 0): type, metric, dim, the creation parameters that decide results, W, each rank
 *                file's row count, size and 64-bit digest, and (IVF_FLAT, IVF_PQ) the digest of the trained state.  Files are
 *                written under temporary names and renamed into place only when every rank has written its own; a failed
 *                save (EINTERNAL) leaves an earlier snapshot under the same prefix as it was.
 *   shard_load : restores a snapshot into this shard's indexes, which must be empty (else EILLEGAL_PARAMETERS); a list-sharded
 *                index may already be trained, with the snapshot's state.  The manifest, every rank file's size and digest
 *                and (same world) the owner of every row are checked before any index changes: a missing, truncated,
 *                swapped or mismatched file, or an index that does not match the manifest -> EINTERNAL, every index left
 *                empty and loadable.  Same world W: rank r restores file r, and its lists, rows and trained state equal the
 *                saved rank's byte for byte.  Another world W' (FLAT, IVF_FLAT, IVF_PQ): every rank installs the trained
 *                state, file f is read by rank f mod W', and every row travels to its owner under W' through shard_add's
 *                routing (rank 0's rows first) with its saved list, stored exactly as saved: no re-assignment, no second
 *                cosine normalisation, IVF_PQ codes never re-encoded.  HNSW onto W' != W: EVECTOR_NOT_SUPPORT.
 *
 * Binary shards (DESIGN.md 4.5): BINARY_IVF_FLAT is sharded by list like IVF_FLAT, BINARY_FLAT by row like FLAT.  They are
 * created and fed through the _binary family below, on packed rows and queries of dim / 8 bytes (as b200vs_add_with_ids_binary);
 * shard_destroy, shard_list_range, shard_broadcast_state (the 'IVFB' state), shard_remove_ids, shard_save, shard_load and
 * b200vs_row_owner serve both kinds.  On a binary shard:
 *   shard_create_binary : BINARY_IVF_FLAT (untrained or trained, as IVF_FLAT) or an EMPTY BINARY_FLAT; a float index:
 *                     EILLEGAL_PARAMETERS.  shard_create keeps refusing binary indexes (EVECTOR_NOT_SUPPORT)
 *   the float data calls (train, add[_device], search[_device], range_search[_device]): EILLEGAL_PARAMETERS, and the _binary
 *                     ones on a float shard too (a refused read still uses up its sequence number); shard_plan_add_device
 *                     and shard_plan_commit: EVECTOR_NOT_SUPPORT; shard_hnsw_add_batched: EILLEGAL_PARAMETERS
 *   shard_train_binary : BINARY_IVF_FLAT: shard_train's flow with b200vs_train_binary's k-means on each rank's rows (nlist / world
 *                     packed centroids each, one all-gather); at world = 1 the state equals b200vs_train_binary's.  BINARY_FLAT: OK
 *   shard_add_binary[_device] : BINARY_IVF_FLAT: the sender assigns each row with the Hamming coarse pass (nearest list, ties to
 *                     the smaller list id) and the packed row travels to the list's owner; BINARY_FLAT: rows travel to
 *                     b200vs_row_owner(id), an id repeated in the collective call -> EVECTOR_ID_DUPLICATED on every rank
 *   shard_search_binary[_device] : BINARY_IVF_FLAT: Hamming coarse pass on the rank's slice + all-gather of the probe table, then
 *                     the binary list scan (BMMA tile scan or exact Hamming scan, as b200vs_search_binary chooses) of the owned
 *                     probed lists; BINARY_FLAT: the rank's own rows.  The merge key is the Hamming distance, which is also the
 *                     API distance.  Results equal b200vs_search_binary on the unsharded index bit for bit.
 *   shard_range_search_binary[_device] : b200vs_range_search_binary's rule (radius clamped to dim + 1 and truncated, hits have
 *                     distance < radius), equal bit for bit; a NaN radius: EILLEGAL_PARAMETERS on every rank before the first
 *                     collective (its sequence number is used up).
 * Snapshots of binary shards are rank files in b200vs_save's "B2VSBIN1" container; both kinds restore onto another world. */
#define B200VS_SHARD_ID_BYTES 128
typedef struct b200vs_shard b200vs_shard;
int b200vs_shard_unique_id(uint8_t id[B200VS_SHARD_ID_BYTES]);
int b200vs_shard_create(b200vs_index* idx, int32_t rank, int32_t world, const uint8_t id[B200VS_SHARD_ID_BYTES], int32_t lanes,
                        b200vs_shard** out);
void b200vs_shard_destroy(b200vs_shard* shard);
int b200vs_shard_list_range(b200vs_shard* shard, int32_t rank, int32_t* begin, int32_t* end);
int b200vs_shard_train(b200vs_shard* shard, int64_t n, const float* x);
int b200vs_shard_broadcast_state(b200vs_shard* shard, int32_t root);
int b200vs_shard_add(b200vs_shard* shard, int64_t n, const float* x, const int64_t* ids);
int b200vs_shard_add_device(b200vs_shard* shard, int64_t n, const float* x_dev, const int64_t* ids_dev);
/* collective Delete: every rank passes the same ids; *n_removed = rows removed over all ranks; EVECTOR_INVALID when no rank held
 * any of them (vector_index_ivf_flat.cc:180-184; row-sharded FLAT / HNSW: OK).  shard_add* appends
 * (IndexIVFFlat::add_with_ids); an Upsert is this call (a not-found status ignored) followed by shard_add*. */
int b200vs_shard_remove_ids(b200vs_shard* shard, int64_t n, const int64_t* ids, int64_t* n_removed);
/* collective batched HNSW build of a row-sharded HNSW index (see above); batch as b200vs_hnsw_add_batched */
int b200vs_shard_hnsw_add_batched(b200vs_shard* shard, int64_t n, const float* x, const int64_t* ids, int32_t batch);
/* owner rank of each id in a row-sharded index of `world` ranks: splitmix64's finalizer of the id read as a uint64, mod world
 * (z ^= z >> 30; z *= 0xbf58476d1ce4e5b9; z ^= z >> 27; z *= 0x94d049bb133111eb; z ^= z >> 31); world in [1, 1024].  A pure
 * host function: no handle, no GPU.  Callers place rows on their owner so that shard_add moves nothing. */
int b200vs_row_owner(int32_t world, int64_t n, const int64_t* ids, int32_t* out_rank);
/* collective snapshot save / restore of a sharded index (see above) */
int b200vs_shard_save(b200vs_shard* shard, const char* prefix);
int b200vs_shard_load(b200vs_shard* shard, const char* prefix);

/* Rebuilds of a sharded set (DESIGN.md 4.9).  Both calls are collectives of the write path, like shard_save / shard_load: every
 * rank calls them in the same order relative to the other writes of that shard, they use up no search sequence number, and
 * every rank returns the same status.
 *
 * shard_need_rebuild: b200vs_need_rebuild's rule applied to the figures of the whole set (one all-gather of every rank's live
 * and tombstoned rows), 1 = rebuild, 0 = not, < 0 = a status negated.  train_rows_set is kept in the shard handle, not in the
 * rank indexes (each rank index's own b200vs_need_rebuild answers as before): the rows shard_train[_binary] clustered over
 * every rank, or every rank's live rows summed at shard_broadcast_state and shard_load, or the rows shard_rebuild_from
 * trained dst on; it is not saved.
 *   IVF_FLAT, BINARY_IVF_FLAT : untrained, or created with nlist 1: 0; else sum(live) >= 256 * nlist and
 *                               train_rows_set <= sum(live) / 2 (shard_train never degenerates nlist: it refuses)
 *   IVF_PQ                    : sum(live) / 2 >= train_rows_set; untrained: 0 (a set is always in IVF-PQ mode)
 *   HNSW                      : sum(deleted) > 0 and sum(deleted) > (sum(live) + sum(deleted)) / 2
 *   FLAT, BINARY_FLAT         : 0
 *
 * shard_rebuild_from: every rank passes its own dst and src.  dst is a fresh shard (shard_create[_binary] under its own unique
 * id) of the same world and rank, with an empty (IVF types: untrained) index of src's type, metric, dimension, nlist,
 * nsubvector, nbits, nlinks, efconstruction and device.  *n_rows (nullable) = the live rows this rank's dst holds afterwards.
 *   IVF_FLAT, BINARY_IVF_FLAT (by list) : let rows_r be src's live rows with b200vs_row_owner(id, world) == r in ascending id
 *                     order (ties: by src rank, then that rank's list-major export order), taken as stored (cosine rows are
 *                     not normalised again).  dst ends up equal, byte for byte (trained state, every list's ids and rows, the
 *                     FP16 mirror), to a fresh shard on which every rank r called shard_train[_binary](rows_r) and then
 *                     shard_add[_binary](rows_r, ids_r).  Routing the training rows by row_owner keeps the rank-local k-means
 *                     balanced whatever the old list layout.  At world 1 this equals b200vs_rebuild_from.  No row crosses
 *                     PCIe: src's live rows are sorted and routed on the device over dst's write stream and communicator.
 *   HNSW (by row)   : each rank runs b200vs_rebuild_from of its src index into its dst index; nothing moves between ranks.
 *   FLAT, BINARY_FLAT, IVF_PQ : EVECTOR_NOT_SUPPORT on every rank (an IVF_PQ set stores only codes: rebuild it from host
 *                     rows with shard_train + shard_add).
 * EILLEGAL_PARAMETERS, on every rank when any rank meets it (the first in rank order), before any index changes: a different
 * world or rank, a dst that is not empty or (IVF types) already trained, differing creation parameters, an HNSW dst whose
 * max_elements is below its rank's live rows, and a rank that would receive fewer than nlist / world training rows
 * (shard_train's refusal; the rule never asks for a rebuild then).  dst == src is refused on the rank that passes it, before
 * any collective, so every rank must pass it alike.  An src with no live rows on any rank: OK, dst stays untrained, *n_rows
 * = 0.  A device failure after the agreement: EINTERNAL on every rank, src unchanged, dst to be discarded.
 * Locks: src's writes wait for the call, its reads (shard_search, deep, range, on src's own lanes and communicators) go on
 * and return unchanged results; none of src's communicators is used.  dst's writes wait too.
 * Peak device memory per rank (by list): src's rows, plus about three copies of this rank's share of the live rows while
 * they are sorted and routed (the sorted local copy, the partitioned send copy, the received copy; the local copy is freed
 * once routed), then the training copy rows_r, shard_add's partitioned and received copies of it (cosine: and its
 * normalised copy) and dst's rows.
 *
 * shard_rebuild_from_range: the split and merge rebuilds of a region served by a sharded set (b200vs_rebuild_from_range's
 * counterpart).  Every rank passes its own dst and its own rank's shards of the n_src source sets; dst is a fresh shard as
 * for shard_rebuild_from, of the same world and rank as every source.  R = the union, over every source set and every rank
 * of it, of the live rows with id_min <= id < id_max (id_max exclusive).  *n_rows (nullable) = the live rows this rank's dst
 * holds afterwards.
 *   IVF_FLAT, BINARY_IVF_FLAT (by list) : rows_r = the rows of R with b200vs_row_owner(id, world) == r in ascending id order
 *                     (ties inside one source set: by source rank, then that rank's list-major export order), taken as stored
 *                     (cosine rows are not normalised again).  dst ends up equal, byte for byte (trained state, every list's
 *                     ids and rows, the FP16 mirror), to a fresh set on which every rank r called shard_train[_binary](rows_r)
 *                     and then shard_add[_binary](rows_r, ids_r).  No row crosses PCIe: each source set's rows in the range are
 *                     sorted and routed to their owner in turn, then what arrived is sorted by id on the owner, with each
 *                     row's source set carried in the sort's value, on dst's write stream and communicator.
 *   FLAT, BINARY_FLAT, HNSW (by row) : every row already sits on row_owner(id, world): each rank runs b200vs_rebuild_from_range
 *                     of its sources' rank indexes into its dst index, and nothing moves between ranks (HNSW: levels from
 *                     dst's fresh generator, no tombstones).
 *   IVF_PQ          : EVECTOR_NOT_SUPPORT on every rank (the set stores only codes).
 * With one source and [0, INT64_MAX) the result equals shard_rebuild_from's on every type that call serves; at world 1 it
 * equals b200vs_rebuild_from_range of the rank-0 indexes.  An empty R (id_min == id_max included): OK, dst stays untrained and
 * *n_rows = 0 on every rank.  dst's training size for shard_need_rebuild becomes the sum of |rows_r|.
 * EILLEGAL_PARAMETERS, on every rank when any rank meets it (the first in rank order), before any index changes: id_min >
 * id_max, a source of another world or rank than dst, a source that differs from dst in type, metric, dimension, nlist,
 * nlinks, efconstruction or device, a dst that is not empty or (IVF types) already trained, an HNSW dst whose max_elements
 * is below its rank's share of R, and a rank that would receive fewer than nlist / world training rows.
 * EVECTOR_ID_DUPLICATED, on every rank, before dst changes: an id live in more than one source set (a split's or merge's
 * sources hold disjoint ranges); copies of one id inside one source set stay legal.  By list, the copies of an id can sit on
 * different ranks, so the check runs after the routing, where every copy of an id meets on its owner.
 * Refused on the rank that meets them, before any collective (every rank must pass them alike): n_src outside [1, 16], a
 * null srcs or null entry, dst among the sources, a source listed twice.  A device failure after the agreement: EINTERNAL on
 * every rank, the sources unchanged, dst to be discarded.
 * Concurrency: a set's writes hold its write gate exclusively; a rebuild holds dst's gate exclusively and every source set's
 * gate shared, all taken in one order (by handle address), and a shared hold is granted whenever no write holds the gate,
 * even while a write waits for it.  So a source set's writes wait for the call, and its reads (shard_search, deep and range
 * searches, on its own lanes and communicators) go on and return unchanged results; none of the sources' communicators is
 * used.  Rebuilds that read the same source sets (a split's child and parent, a merge beside a split of one of its sources)
 * never wait for each other's locks on a rank, whatever order they start in.  That does not make their collectives safe to
 * interleave: each rebuild runs its collectives on its own dst communicator and allocates and frees device memory between
 * them, and cudaFree synchronises the device, so on NCCL over real GPUs one rebuild's free can wait for another's collective
 * kernel, which waits for a peer rank stuck the same way the other way round.  So on NCCL run a rank's rebuilds one after
 * another, in the same order on every rank (a split: the child, then the parent); run them at once only over a collective
 * library whose ranks meet on the host.  A write to a source set and the rebuilds that read it: every rank must order them
 * the same way, and a write meant to follow a rebuild must be issued only after that rebuild has returned on its rank (a
 * write that waits for a gate held shared can be overtaken by a rebuild issued after it; a steady stream of overlapping
 * rebuilds would keep a source's writes waiting).
 * Peak device memory per rank (by list): the sources' rows, plus, one source set at a time, its sorted local copy of the
 * range, the partitioned send copy and the received copy (the local copy is freed once routed); then every source set's
 * received copy at once with 16 B per row of sort keys and values (the value carries the row's source set in its top bits)
 * and 16 B per row of sorted output, then the training copy rows_r, shard_add's partitioned and received copies of it
 * (cosine: and its normalised copy) and dst's rows. */
int b200vs_shard_need_rebuild(b200vs_shard* shard);
int b200vs_shard_rebuild_from(b200vs_shard* dst, b200vs_shard* src, int64_t* n_rows);
int b200vs_shard_rebuild_from_range(b200vs_shard* dst, int32_t n_src, b200vs_shard* const* srcs, int64_t id_min, int64_t id_max,
                                    int64_t* n_rows);
int b200vs_shard_plan_add_device(b200vs_shard* shard, int64_t n, const float* x_dev);
int b200vs_shard_plan_commit(b200vs_shard* shard);
int b200vs_shard_search(b200vs_shard* shard, int64_t seq, int64_t nq, const float* xq, int32_t k, const b200vs_search_params* sp,
                        float* out_dist, int64_t* out_ids);
int b200vs_shard_search_device(b200vs_shard* shard, int64_t seq, int64_t nq, const float* xq_dev, int32_t k,
                               const b200vs_search_params* sp, float* out_dist_dev, int64_t* out_ids_dev, void* stream);
/* shard_search_deep / shard_search_binary_deep: b200vs_search_deep / b200vs_search_binary_deep over the sharded index, for
 * any k in [1, B200VS_DEEP_MAX_K].  Host pointers; collective reads in shard_search's flow (same sequence numbers, lanes and
 * communicators: deep, top-k and range batches may be interleaved).  Types: list-sharded IVF_FLAT, IVF_PQ and
 * BINARY_IVF_FLAT, row-sharded FLAT and BINARY_FLAT.  Each rank runs the deep path on its lists or rows, keyed the way the
 * single-index deep path orders its output (L2 distance | -ip | Hamming distance, then id); the per-rank sorted runs are
 * all-gathered one query chunk at a time (at most 1 GiB of 16-byte records per chunk on each rank) and merged by a pairwise
 * merge tree with no shared-memory bound on k (DESIGN.md 4.5, 4.10).  Results (distances, ids, -1 / 0 padding) equal
 * b200vs_search_deep / b200vs_search_binary_deep bit for bit on one unsharded index holding every rank's rows with the same
 * trained state, and b200vs_shard_search wherever that answers.  Refused on every rank before the first collective, a refused
 * call still using up its sequence number: k > B200VS_DEEP_MAX_K, null outputs, a float call on a binary shard or the
 * reverse, and (IVF_PQ) a LUT alone larger than one SM's shared memory: EILLEGAL_PARAMETERS; row-sharded HNSW:
 * EVECTOR_NOT_SUPPORT.  k <= 0: OK, nothing done.  b200vs_last_search_stats[0] counts the call's launches; with profiling
 * on, phase slots [10] (collectives) and [11] (pack + merge) are filled as for shard_search. */
int b200vs_shard_search_deep(b200vs_shard* shard, int64_t seq, int64_t nq, const float* xq, int32_t k, const b200vs_search_params* sp,
                             float* out_dist, int64_t* out_ids);
int b200vs_shard_search_binary_deep(b200vs_shard* shard, int64_t seq, int64_t nq, const uint8_t* xq, int32_t k,
                                    const b200vs_search_params* sp, float* out_dist, int64_t* out_ids);
/* shard_range_search[_device]: b200vs_range_search over the sharded index, in shard_search's flow (same sequence numbers,
 * lanes and communicators: range and top-k batches may be interleaved).  Step 2 is the range scan of the owned probed lists
 * (IVF_FLAT: the tile range scan; IVF_PQ: the thresholded LUT scan); the all-gathered payload is nq * max_results * 16 bytes
 * per rank; the merge orders hits as the single-index select does (L2 distance | -ip, then id).  Results (distances, ids and
 * counts) equal b200vs_range_search on the unsharded index.  Refused on every rank before the first collective: max_results
 * outside [1, 4096], null outputs, and (IVF_PQ) a LUT + select pool larger than one SM's shared memory; a refused call still
 * uses up its sequence number.  A NaN radius is not refused: every rank contributes no hits and the call returns empty
 * results, as b200vs_range_search does. */
int b200vs_shard_range_search(b200vs_shard* shard, int64_t seq, int64_t nq, const float* xq, float radius, int32_t max_results,
                              const b200vs_search_params* sp, float* out_dist, int64_t* out_ids, int32_t* out_counts);
int b200vs_shard_range_search_device(b200vs_shard* shard, int64_t seq, int64_t nq, const float* xq_dev, float radius,
                                     int32_t max_results, const b200vs_search_params* sp, float* out_dist_dev,
                                     int64_t* out_ids_dev, int32_t* out_counts_dev, void* stream);
/* binary shards (see above): packed rows and queries, dim / 8 bytes each */
int b200vs_shard_create_binary(b200vs_index* idx, int32_t rank, int32_t world, const uint8_t id[B200VS_SHARD_ID_BYTES],
                               int32_t lanes, b200vs_shard** out);
int b200vs_shard_train_binary(b200vs_shard* shard, int64_t n, const uint8_t* x);
int b200vs_shard_add_binary(b200vs_shard* shard, int64_t n, const uint8_t* x, const int64_t* ids);
int b200vs_shard_add_binary_device(b200vs_shard* shard, int64_t n, const uint8_t* x_dev, const int64_t* ids_dev);
int b200vs_shard_search_binary(b200vs_shard* shard, int64_t seq, int64_t nq, const uint8_t* xq, int32_t k,
                               const b200vs_search_params* sp, float* out_dist, int64_t* out_ids);
int b200vs_shard_search_binary_device(b200vs_shard* shard, int64_t seq, int64_t nq, const uint8_t* xq_dev, int32_t k,
                                      const b200vs_search_params* sp, float* out_dist_dev, int64_t* out_ids_dev, void* stream);
int b200vs_shard_range_search_binary(b200vs_shard* shard, int64_t seq, int64_t nq, const uint8_t* xq, float radius,
                                     int32_t max_results, const b200vs_search_params* sp, float* out_dist, int64_t* out_ids,
                                     int32_t* out_counts);
int b200vs_shard_range_search_binary_device(b200vs_shard* shard, int64_t seq, int64_t nq, const uint8_t* xq_dev, float radius,
                                            int32_t max_results, const b200vs_search_params* sp, float* out_dist_dev,
                                            int64_t* out_ids_dev, int32_t* out_counts_dev, void* stream);

/* Device-pointer write path of a single index (IVF_FLAT, IVF_PQ in its IVF-PQ mode): rows and ids already on the index's
 * device.  lists_dev (nullable) = the inverted list of every row when the caller has already assigned them
 * (b200vs_assign_device); returns when done.  IVF_PQ: codes, ids and list layout equal a host b200vs_add_with_ids's. */
int b200vs_add_with_ids_device(b200vs_index* idx, int64_t n, const float* x_dev, const int64_t* ids_dev, const int64_t* lists_dev,
                               int upsert);
/* faiss quantizer->assign: nearest centroid of every (raw) row, out_lists_dev[n]; synchronous. */
int b200vs_assign_device(b200vs_index* idx, int64_t n, const float* x_dev, int64_t* out_lists_dev);
/* Pre-size every inverted list of an EMPTY trained IVF_FLAT or IVF_PQ index (rows_per_list[nlist], host) in one arena
 * allocation. */
int b200vs_reserve_lists(b200vs_index* idx, const int64_t* rows_per_list, int32_t nlist);

/* Pairwise distance matrix, the UtilService path UtilServiceImpl::VectorCalcDistance (src/server/util_service.cc:45-92)
 * -> VectorIndexUtils::CalcDistanceEntry / CalcDistanceCore (src/vector/vector_index_utils.cc:48-124).  Host pointers,
 * row-major left [nl, dim], right [nr, dim]; out [nl, nr]: L2 -> squared L2, IP -> 1 - ip, COSINE -> 1 - ip of the
 * normalised copies (algorithm FAISS: NormalizeVectorForFaiss :480-491; HNSWLIB: NormalizeVectorForHnsw :493-500).
 * left_out / right_out (nullable) = what is_return_normlize returns: the normalised copies for COSINE, else the inputs. */
enum { B200VS_ALGORITHM_FAISS = 1, B200VS_ALGORITHM_HNSWLIB = 2 };  /* pb::index::AlgorithmType */
int b200vs_calc_distance(int32_t device, int32_t algorithm, b200vs_metric metric, int32_t dim, int64_t nl, const float* left,
                         int64_t nr, const float* right, float* out, float* left_out, float* right_out);
/* The same matrix for METRIC_TYPE_HAMMING (CalcHammingDistanceByFaiss, vector_index_utils.cc:333-357).  Host pointers,
 * packed rows left [nl, nbytes], right [nr, nbytes]; out [nl, nr] = popcount(left_i XOR right_j) over the nbytes bytes,
 * as float (an exact integer).  nbytes <= 0 or > 4096 (32768 bits, the binary index limit): EILLEGAL_PARAMETERS; then
 * nl == 0 or nr == 0 returns OK and computes nothing. */
int b200vs_calc_distance_binary(int32_t device, int32_t nbytes, int64_t nl, const uint8_t* left, int64_t nr, const uint8_t* right,
                                float* out);

/* Streaming brute-force search over vectors that are NOT in an index: VectorReader::BruteForceSearch
 * (src/vector/vector_reader.cc:1873-2048), which scans the region's vector column family, builds a temporary Flat
 * index per FLAGS_vector_index_bruteforce_batch_count vectors, searches it and keeps per-query top-k heaps.
 *   scan_begin : the queries (host, raw; COSINE is normalised inside), k, optional id filters (copied);
 *   scan_push  : one tile of scanned vectors + ids (host; any size, ids unique inside a tile) -> tile top-k on the GPU,
 *                merged into the running top-k with the (distance, id) rule;
 *   scan_finish: running top-k -> out_dist / out_ids [nq, k] (API distances ascending, -1 padded); frees the handle.
 * The result equals one Flat search over the concatenation of all tiles.  A k past the exact scan's shared-memory select
 * (k > 8192 at small dim, less at large dim) takes each tile's top-k and the merge through the deep path of
 * b200vs_search_deep, up to B200VS_DEEP_MAX_K; a larger one is refused at scan_begin with EILLEGAL_PARAMETERS. */
typedef struct b200vs_scan b200vs_scan;
int b200vs_scan_begin(int32_t device, b200vs_metric metric, int32_t dim, int64_t nq, const float* xq, int32_t k,
                      const b200vs_search_params* sp, b200vs_scan** out);
int b200vs_scan_push(b200vs_scan* scan, int64_t n, const float* x, const int64_t* ids);
int b200vs_scan_finish(b200vs_scan* scan, float* out_dist, int64_t* out_ids);
void b200vs_scan_abort(b200vs_scan* scan);

/* Streaming brute-force RANGE search over vectors that are not in an index: VectorReader::BruteForceRangeSearch
 * (src/vector/vector_reader.cc:2050-2202), which scans the same tiles, range-searches a temporary Flat index per tile with
 * one query per task (vector_index_flat.cc:267-323) and appends each tile's hits per query until
 * FLAGS_vector_index_max_range_search_result_count (later hits are dropped; the reader does not sort).  The rule:
 *   - a row is a hit when its id is >= 0, it passes the filters, and its exact FP32 value (the value b200vs_range_search
 *     computes on a Flat index, bit for bit) is strictly inside the radius: L2 dist < radius; IP / COSINE ip > 1 - radius
 *     (COSINE rows and queries are normalised as a Flat index normalises them);
 *   - per query the result is the FIRST max_results hits in scan order: tiles in push order, rows in their order within a
 *     tile.  Unlike b200vs_range_search, which keeps the closest max_results, nothing is sorted.  The in-tile order is the
 *     storage order a one-query faiss Flat range search visits; that is upstream faiss behaviour, recalled, not pinned
 *     against the reference build;
 *   - distances in API semantics: squared L2, or 1 - ip (FillRangeSearchResult, vector_index_utils.cc:657-694).
 * All pointers are host pointers.
 *   scan_range_begin : argument checks and statuses of b200vs_scan_begin, then max_results <= 0 -> EILLEGAL_PARAMETERS; the
 *                      queries and filters (id range, sorted id list, negate) are copied; a failed allocation returns
 *                      EINTERNAL and no handle; a NaN radius (either sign) admits no row, so its pushes add nothing;
 *   scan_range_push  : one tile (n <= 0: no-op); a repeated id inside the tile -> EVECTOR_ID_DUPLICATED, the tile adds
 *                      nothing and the handle stays usable; returns when the tile has been scanned;
 *   scan_range_finish: out_counts[nq] = hits kept; out_dist / out_ids [nq, max_results] hold them in scan order in slots
 *                      [0, count), then id -1, distance 0.  Frees the handle, also when it fails. */
typedef struct b200vs_scan_range b200vs_scan_range;
int b200vs_scan_range_begin(int32_t device, b200vs_metric metric, int32_t dim, int64_t nq, const float* xq, float radius,
                            int32_t max_results, const b200vs_search_params* sp, b200vs_scan_range** out);
int b200vs_scan_range_push(b200vs_scan_range* scan, int64_t n, const float* x, const int64_t* ids);
int b200vs_scan_range_finish(b200vs_scan_range* scan, float* out_dist, int64_t* out_ids, int32_t* out_counts);
void b200vs_scan_range_abort(b200vs_scan_range* scan);

/* The same brute-force searches answered from an index's own device rows, in place of the RocksDB scan whose rows a reader
 * pushes through b200vs_scan_* / b200vs_scan_range_* (VectorReader::BruteForceSearch / BruteForceRangeSearch, the road of
 * every request with use_brute_force and of every range search on HNSW).  Host pointers; readers, under the index's read
 * lock like b200vs_search.  The result is what b200vs_scan_begin/push/finish (b200vs_scan_range_begin/push/finish) returns
 * when fed the index's live rows in ascending id order with the same queries, k (radius, max_results), metric and sp, bit
 * for bit (ids, distance bits, counts):
 *   - top-k: exact, ordered by (API distance, id), -1 / 0 padded, any k up to B200VS_DEEP_MAX_K (past the exact scan's
 *     select pool through the deep path, as b200vs_scan_* does).  The rows may be fed in any chunking, with one exception
 *     that the chunked scan itself carries under IP / COSINE: where 1 - ip rounds two rows' different ip values to one
 *     distance at the k-th slot, a chunking that splits them may keep the smaller id where one chunk keeps the larger ip;
 *   - range: per query the FIRST max_results hits in ascending id order (RocksDB key order), unsorted.  Rows sharing an id
 *     (an IVF_FLAT add without upsert) come in storage order; the scan takes them in that order in separate chunks, as
 *     b200vs_scan_range_push refuses a repeated id inside one tile.
 * sp's filters apply (id range, sorted id list, negate); nprobe and efsearch are ignored; exact_only is accepted and changes
 * nothing.  Stored cosine rows are not normalised again; the queries are normalised as b200vs_scan_begin does.
 * Types: FLAT, IVF_FLAT (every metric) and HNSW under L2 / IP.  IVF_PQ (codes only), BINARY_FLAT, BINARY_IVF_FLAT and HNSW
 * under COSINE (its rows carry NormalizeVectorForHnsw's bits, which a scan over raw rows does not reproduce):
 * EVECTOR_NOT_SUPPORT, nothing launched, the index unchanged; the caller keeps its RocksDB scan.
 * An empty or untrained index: empty results.  k <= 0: OK, nothing done; k > B200VS_DEEP_MAX_K, max_results <= 0 or a null
 * output: EILLEGAL_PARAMETERS.  A NaN radius admits no row: every count 0, nothing launched.  No row is copied: top-k scans
 * the rows in place (tombstones, unused slots and deleted nodes count as id -1 through a per-call id view); range compacts
 * the live rows that pass the filters into a row list, sorts it by id and walks the rows through it. */
int b200vs_brute_force_search(b200vs_index* idx, int64_t nq, const float* xq, int32_t k, const b200vs_search_params* sp,
                              float* out_dist, int64_t* out_ids);
int b200vs_brute_force_range_search(b200vs_index* idx, int64_t nq, const float* xq, float radius, int32_t max_results,
                                    const b200vs_search_params* sp, float* out_dist, int64_t* out_ids, int32_t* out_counts);

/* Counters of the last search on this index: [0] kernels launched, [1] queries served by the tensor-core
 * candidate pass; with profiling on (b200vs_set_profiling) also [2] queries of the tensor-core pass that failed
 * certification and were re-run on the exact path (0 with profiling off), [3] device time of the dominant list-scan
 * kernel in ns (CUDA events on the launch stream), [4] rows in the distinct probed lists, [5] distinct probed lists,
 * [6] work items of the tile scan, [7] its tensor-core work (128-row tiles x padded query columns).  Binary indexes
 * keep these meanings for their BMMA tile scan: [1] queries it served, [2] queries re-run on the exact Hamming scan
 * (capture overflow, or fewer than k eligible sampled rows), [3] its capture kernel.  HNSW fills [0] and
 * [6] = queries walked with the candidate-heap form (id filter, tombstones or ef >= 1024; 0 = merged-array form).  Profiling
 * synchronises the stream inside the call: never leave it on in a timed run. */
int b200vs_last_search_stats(b200vs_index* idx, int64_t stats[8]);
/* With profiling on: device milliseconds (CUDA events on the launch stream) the last search spent in each phase of the
 * IVF tile path (binary tile scans fill [3]-[9] the same way; [7] is their final select): [0] coarse prep, [1] coarse scan, [2] coarse select + exact re-score, [3] work planning + query
 * gather, [4] sample pass, [5] thresholds, [6] list scan (capture), [7] final select + exact re-score, [8] exact
 * fallback for uncertified queries, [9] other, [10] collectives of a sharded search (b200vs_shard_search*), [11] pack + merge of
 * the per-shard top-k.  After b200vs_hnsw_add_batched: [12] construction search, [13] peer distances + forward links,
 * [14] reverse links, summed over the call's batches.  Unused slots are 0. */
int b200vs_last_phase_times(b200vs_index* idx, float ms[16]);
int b200vs_set_profiling(b200vs_index* idx, int on);

/* Diagnostics (tests only): the tile kernel's approximate scores of a FLAT index's rows.  split = 0: list-scan
 * arithmetic without an FP16 mirror (rows truncated by the tensor core, queries rounded to TF32); split = 1: the coarse
 * pass's hi/lo arithmetic; split = 2: the list scan on an IVF-Flat FP16 mirror (rows and queries scaled by powers of two
 * and rounded to FP16; needs dim % 8 == 0).  split = 3 / 4: the threshold sample pass's scores in the arithmetic of
 * split = 0 / 2, from the tile kernel's sample configuration, for the rows it samples (the first 32 rows of every
 * 2048-row span, with the index as one list); every other row is NaN.  xq [nq, dim] RAW (normalised inside for COSINE, as search does); out_scores [nq, rows] with rows =
 * count + deleted count in storage order (L2: ||x||^2 - 2<q,x>; IP / cosine: -<q,x>; tombstoned rows +inf);
 * out_eps [nq] = the tc_eps() value the finish kernels use for that query and mode.  Non-FLAT indexes, dim % 4 != 0,
 * dim < 32, split = 2 or 4 with dim % 8 != 0 and any other split value: EILLEGAL_PARAMETERS. */
int b200vs_debug_tc_scores(b200vs_index* idx, int64_t nq, const float* xq, int32_t split, float* out_scores, float* out_eps);

const char* b200vs_last_error(void);
const char* b200vs_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B200VS_H_ */
