// vector_index_b200.h — drop-in subclass of dingodb::VectorIndex backed by libb200vs (include/b200vs.h).
//
// One class serves the six plugin types; VectorIndexFactory::New{Flat,IvfFlat,IvfPq,Hnsw,BinaryFlat,BinaryIvfFlat}
// (src/vector/vector_index_factory.cc:40-95) would return it instead of VectorIndexFlat / VectorIndexIvfFlat /
// VectorIndexIvfPq / VectorIndexHnsw and their faiss::IndexBinary instantiations.  Binary types hold packed UINT8
// vectors (binary_values, dimension in bits) under METRIC_TYPE_HAMMING.  The class does only what the reference plugins
// do around their faiss / hnswlib calls: argument checks with the same status codes, pb -> flat-array marshalling
// (CheckVectorDimension / ExtractVectorValue / FillSearchResult, src/vector/vector_index_utils.cc:502-655), filter
// lowering, and the write lock bookkeeping; all arithmetic is behind the C ABI.
#pragma once
#ifdef B200VS_WITH_DINGO_HEADERS
#include "vector/vector_index.h"
#else
#include "dingo_shim.h"
#endif

#include <atomic>
#include <shared_mutex>
#include <string>
#include <vector>

#include "../../include/b200vs.h"

namespace dingodb {

class VectorIndexB200 : public VectorIndex {
 public:
  VectorIndexB200(int64_t id, const pb::common::VectorIndexParameter& vector_index_parameter, const pb::common::RegionEpoch& epoch,
                  const pb::common::Range& range, ThreadPoolPtr thread_pool, int device = 0);
  ~VectorIndexB200() override;

  VectorIndexB200(const VectorIndexB200&) = delete;
  VectorIndexB200& operator=(const VectorIndexB200&) = delete;

  int32_t GetDimension() override { return dimension_; }
  pb::common::MetricType GetMetricType() override { return metric_type_; }
  butil::Status GetCount(int64_t& count) override;
  butil::Status GetDeletedCount(int64_t& deleted_count) override;
  butil::Status GetMemorySize(int64_t& memory_size) override;
  bool IsExceedsMaxElements(int64_t vector_size) override;

  butil::Status Add(const std::vector<pb::common::VectorWithId>& vector_with_ids) override;
  butil::Status Upsert(const std::vector<pb::common::VectorWithId>& vector_with_ids) override;
  butil::Status Delete(const std::vector<int64_t>& delete_ids) override;

  butil::Status Save(const std::string& path) override;
  butil::Status Load(const std::string& path) override;

  butil::Status Search(const std::vector<pb::common::VectorWithId>& vector_with_ids, uint32_t topk,
                       const std::vector<std::shared_ptr<FilterFunctor>>& filters, bool reconstruct,
                       const pb::common::VectorSearchParameter& parameter,
                       std::vector<pb::index::VectorWithDistanceResult>& results) override;
  butil::Status RangeSearch(const std::vector<pb::common::VectorWithId>& vector_with_ids, float radius,
                            const std::vector<std::shared_ptr<FilterFunctor>>& filters, bool reconstruct,
                            const pb::common::VectorSearchParameter& parameter,
                            std::vector<pb::index::VectorWithDistanceResult>& results) override;

  // With support_fork_save, LockWrite also stages the snapshot (b200vs_save_stage) and UnlockWrite frees it
  void LockWrite() override;
  void UnlockWrite() override;
  butil::Status Train(std::vector<float>& train_datas) override;
  butil::Status Train(std::vector<uint8_t>& train_datas) override;  // packed rows, dimension / 8 bytes each
  butil::Status Train(const std::vector<pb::common::VectorWithId>& vectors) override;
  bool NeedToRebuild() override;  // b200vs_need_rebuild: the reference plugin's rule for this type
  // Fills this fresh index from old's live rows on the GPU (b200vs_rebuild_from), in place of RebuildVectorIndex's RocksDB
  // scan, Train and Add: the result equals a train + add of old's rows in ascending id order.  old keeps serving reads.
  butil::Status RebuildFrom(VectorIndexB200& old);
  // Fills this fresh index from the rows with min_vector_id <= id < max_vector_id of olds (b200vs_rebuild_from_range): the
  // rebuilds of a region split (olds = {share index} for the child, {own index} for the parent) or merge ({own, sibling}).
  // The caller passes the region's range as VectorCodec::DecodeRangeToVectorId gives it.  The olds keep serving reads.
  butil::Status RebuildFrom(const std::vector<VectorIndexB200*>& olds, int64_t min_vector_id, int64_t max_vector_id);
  // VectorReader::BruteForceSearch / BruteForceRangeSearch answered from this index's own device rows
  // (b200vs_brute_force_search / b200vs_brute_force_range_search) instead of the region's RocksDB rows: the filters are
  // lowered as Search lowers them, plus the region's range min_vector_id <= id < max_vector_id (as
  // VectorCodec::DecodeRangeToVectorId gives it), and results are filled as BruteForceScannerB200 /
  // BruteForceRangeScannerB200 fill them (one entry per query; range: at most max_range_search_result_count hits in
  // ascending id order, unsorted).  EVECTOR_NOT_SUPPORT for IVF_PQ, the binary types and HNSW cosine: the caller keeps its
  // RocksDB loop.  Call them only when this index alone serves the region (no share index, no sibling) and IsReady().
  butil::Status BruteForceSearch(const std::vector<pb::common::VectorWithId>& vector_with_ids, uint32_t topk, int64_t min_vector_id,
                                 int64_t max_vector_id, const std::vector<std::shared_ptr<FilterFunctor>>& filters,
                                 std::vector<pb::index::VectorWithDistanceResult>& results);
  butil::Status BruteForceRangeSearch(const std::vector<pb::common::VectorWithId>& vector_with_ids, float radius, int64_t min_vector_id,
                                      int64_t max_vector_id, const std::vector<std::shared_ptr<FilterFunctor>>& filters,
                                      std::vector<pb::index::VectorWithDistanceResult>& results);
  bool NeedTrain() override;
  bool IsTrained() override;
  // the stock plugins' rules (flat.cc:515-531, ivf_flat.cc:786-802, raw_ivf_pq.cc:533-549, ivf_pq.cc:450-462, hnsw.cc:592-609):
  // no rows (HNSW: no live or deleted node) or untrained: false, else last_save_log_behind > 10000.  False without save support.
  bool NeedToSave(int64_t last_save_log_behind) override;
  // fork()-based saving (vector_index_snapshot_manager.cc:583-608) cannot carry a CUDA context into the child.  Without
  // support_fork_save the plugin reports "no save support" like the DiskANN plugin (vector_index_diskann.cc:267) and the
  // server rebuilds from RocksDB; with it, the save is split at the fork (see support_fork_save).
  bool SupportSave() override { return support_fork_save; }
  pb::common::VectorIndexType VectorIndexSubType() override;  // vector_index.h:238

  // largest result count RangeSearch keeps per query (FLAGS_vector_index_max_range_search_result_count, vector_reader.cc:60)
  static int32_t max_range_search_result_count;
  // HNSW Add / Upsert calls of at least this many rows build the graph on the GPU in batches (b200vs_hnsw_add_batched,
  // library default batch); smaller calls keep the host builder.  0 = off: every call takes the host builder.
  static int64_t hnsw_device_build_min_rows;
  // Snapshots through the fork-based save (default false: no save support, as before).  When true, SupportSave() is true
  // for every type; LockWrite takes the write gate and stages in host memory the bytes Save would write (b200vs_save_stage:
  // the device work runs in the parent, under the gate); Save writes the staged bytes (b200vs_save_staged: no CUDA, no lock,
  // no logging, so the forked child may call it), or calls b200vs_save when nothing is staged; UnlockWrite frees the staged
  // bytes and releases the gate.  Costs one host copy of the region's saved rows while the gate is held.
  static bool support_fork_save;

 private:
  butil::Status AddOrUpsert(const std::vector<pb::common::VectorWithId>& vector_with_ids, bool is_upsert);
  butil::Status ToStatus(int rc) const;
  bool Binary() const {
    return vector_index_type == pb::common::VECTOR_INDEX_TYPE_BINARY_FLAT || vector_index_type == pb::common::VECTOR_INDEX_TYPE_BINARY_IVF_FLAT;
  }

  b200vs_index* index_ = nullptr;
  int32_t dimension_ = 0;
  pb::common::MetricType metric_type_ = pb::common::METRIC_TYPE_NONE;
  std::shared_mutex write_gate_;  // LockWrite/UnlockWrite of the snapshot path; reads and writes lock inside the library
  // what LockWrite's stage left for Save: nothing (b200vs_save), an image, or a failed stage and its message
  enum StageState { kNotStaged, kStaged, kStageFailed };
  std::atomic<int> stage_state_{kNotStaged};
  std::string stage_error_;
};

// VectorIndexUtils::CalcDistanceEntry (src/vector/vector_index_utils.cc:48-76) over the C ABI: same operand meaning
// (algorithm_type = pb::index::AlgorithmType: 1 FAISS, 2 HNSWLIB; metric; is_return_normlize) and the same error codes.
class VectorIndexB200Utils {
 public:
  static butil::Status CalcDistance(int algorithm_type, pb::common::MetricType metric_type, const std::vector<pb::common::Vector>& op_left_vectors,
                                    const std::vector<pb::common::Vector>& op_right_vectors, bool is_return_normlize,
                                    std::vector<std::vector<float>>& distances, std::vector<pb::common::Vector>& result_op_left_vectors,
                                    std::vector<pb::common::Vector>& result_op_right_vectors, int device = 0);

 private:
  static butil::Status CalcHammingDistance(int algorithm_type, const std::vector<pb::common::Vector>& op_left_vectors,
                                           const std::vector<pb::common::Vector>& op_right_vectors, bool is_return_normlize,
                                           std::vector<std::vector<float>>& distances, std::vector<pb::common::Vector>& result_op_left_vectors,
                                           std::vector<pb::common::Vector>& result_op_right_vectors, int device);
};

// The inner loop of VectorReader::BruteForceSearch (src/vector/vector_reader.cc:1873-2048): the caller keeps the RocksDB
// iterator, pushes each decoded batch (FLAGS_vector_index_bruteforce_batch_count vectors) and collects the top-k at the end.
class BruteForceScannerB200 {
 public:
  BruteForceScannerB200(pb::common::MetricType metric_type, int32_t dimension, const std::vector<pb::common::VectorWithId>& vector_with_ids,
                        uint32_t topk, int device = 0);
  ~BruteForceScannerB200();
  BruteForceScannerB200(const BruteForceScannerB200&) = delete;
  BruteForceScannerB200& operator=(const BruteForceScannerB200&) = delete;
  butil::Status Push(const std::vector<pb::common::VectorWithId>& vector_with_id_batch);
  butil::Status Finish(std::vector<pb::index::VectorWithDistanceResult>& results);  // ascending by distance, one entry per query

 private:
  b200vs_scan* scan_ = nullptr;
  butil::Status init_status_;
  pb::common::MetricType metric_type_;
  int32_t dimension_;
  size_t nq_;
  uint32_t topk_;
};

// The inner loop of VectorReader::BruteForceRangeSearch (src/vector/vector_reader.cc:2050-2202), the path that also serves
// every range search of an HNSW index (RangeSearch returns EVECTOR_NOT_SUPPORT there).  Each pushed batch is range-searched
// on the GPU without a temporary index; per query the first VectorIndexB200::max_range_search_result_count hits in scan
// order are kept (batches in push order, rows in batch order), unsorted, as the reader keeps them.  Range and sort functors
// run on the GPU; any other functor is applied on the host in Push, so a row is kept only when every filter passes it.
class BruteForceRangeScannerB200 {
 public:
  BruteForceRangeScannerB200(pb::common::MetricType metric_type, int32_t dimension, const std::vector<pb::common::VectorWithId>& vector_with_ids,
                             float radius, const std::vector<std::shared_ptr<VectorIndex::FilterFunctor>>& filters, int device = 0);
  ~BruteForceRangeScannerB200();
  BruteForceRangeScannerB200(const BruteForceRangeScannerB200&) = delete;
  BruteForceRangeScannerB200& operator=(const BruteForceRangeScannerB200&) = delete;
  butil::Status Push(const std::vector<pb::common::VectorWithId>& vector_with_id_batch);
  butil::Status Finish(std::vector<pb::index::VectorWithDistanceResult>& results);  // scan order, one entry per query

 private:
  b200vs_scan_range* scan_ = nullptr;
  butil::Status init_status_;
  pb::common::MetricType metric_type_;
  int32_t dimension_;
  size_t nq_;
  int32_t cap_;
  std::vector<std::shared_ptr<VectorIndex::FilterFunctor>> host_filters_;  // the functors the GPU form cannot express
};

}  // namespace dingodb
