// test_plugin_binary.cc — the drop-in subclass serving VECTOR_INDEX_TYPE_BINARY_FLAT and _BINARY_IVF_FLAT, case by case
// after the reference's gtest suites (test/unit_test/vector/test_vector_index_binary_{flat,ivf_flat}.cc): status codes,
// result counts, value type and metric of every hit, filter containment, training, persistence, and CalcDistance with
// METRIC_TYPE_HAMMING.  Every plugin search is also compared with a direct b200vs_search_binary /
// b200vs_range_search_binary call on an index built from the same rows, so the check covers the marshalling as well.
// Needs a GPU; run by tests/test_gpu_plugin_binary.py.
#include <unistd.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <set>
#include <string>

#include "vector_index_b200.h"

using namespace dingodb;
using Results = std::vector<pb::index::VectorWithDistanceResult>;

static int g_fail = 0;
#define EXPECT(cond)                                                                \
  do {                                                                              \
    if (!(cond)) { ++g_fail; printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); } \
  } while (0)

static std::vector<uint8_t> random_rows(int n, int nb, unsigned seed) {
  std::mt19937 rng(seed);
  std::vector<uint8_t> x((size_t)n * nb);
  for (auto& b : x) b = (uint8_t)(rng() & 0xFF);
  return x;
}
static pb::common::Vector binary_vector(const uint8_t* row, int nb, int dim) {
  pb::common::Vector v;
  v.set_dimension(dim);
  v.set_value_type(pb::common::ValueType::UINT8);
  for (int j = 0; j < nb; ++j) v.add_binary_values(std::string(1, (char)row[j]));
  return v;
}
static std::vector<pb::common::VectorWithId> to_pb(const std::vector<uint8_t>& x, int n, int dim, int64_t first_id) {
  const int nb = dim / 8;
  std::vector<pb::common::VectorWithId> out(n);
  for (int i = 0; i < n; ++i) {
    out[i].set_id(first_id + i);
    *out[i].mutable_vector() = binary_vector(x.data() + (size_t)i * nb, nb, dim);
  }
  return out;
}
static VectorIndexPtr make(pb::common::VectorIndexType t, pb::common::MetricType m, int dim, int nlist = 0) {
  pb::common::VectorIndexParameter p;
  p.set_vector_index_type(t);
  if (t == pb::common::VECTOR_INDEX_TYPE_BINARY_FLAT) { auto* q = p.mutable_binary_flat_parameter(); q->dimension_ = dim; q->metric_type_ = m; }
  if (t == pb::common::VECTOR_INDEX_TYPE_BINARY_IVF_FLAT) { auto* q = p.mutable_binary_ivf_flat_parameter(); q->dimension_ = dim; q->metric_type_ = m; q->ncentroids_ = nlist; }
  if (t == pb::common::VECTOR_INDEX_TYPE_FLAT) { auto* q = p.mutable_flat_parameter(); q->dimension_ = dim; q->metric_type_ = m; }
  return std::make_shared<VectorIndexB200>(1, p, pb::common::RegionEpoch(), pb::common::Range(), nullptr);
}
static VectorIndexPtr make_ok(pb::common::VectorIndexType t, int dim, int nlist = 0) {
  auto ix = make(t, pb::common::METRIC_TYPE_HAMMING, dim, nlist);
  int64_t c = 0;
  if (!ix->GetCount(c).ok()) {  // no CUDA device / library failure: the product has no CPU fallback, so neither has this test
    printf("cannot create the index: %s\n", b200vs_last_error());
    exit(2);
  }
  return ix;
}

// The same rows in an index driven through the C ABI directly.
struct Direct {
  b200vs_index* h = nullptr;
  int nb;
  Direct(b200vs_type t, int dim, int nlist) : nb(dim / 8) {
    b200vs_params p{};
    p.nlist = nlist;
    EXPECT(b200vs_create(t, B200VS_HAMMING, dim, &p, &h) == B200VS_OK);
  }
  ~Direct() { b200vs_destroy(h); }
  // the plugin's results for queries xq equal a direct search (distances as is, ids, count)
  void expect_search(const Results& got, const std::vector<uint8_t>& xq, int nq, int k, int nprobe) {
    b200vs_search_params sp{};
    sp.nprobe = nprobe;
    std::vector<float> D((size_t)nq * k);
    std::vector<int64_t> I((size_t)nq * k);
    EXPECT(b200vs_search_binary(h, nq, xq.data(), k, &sp, D.data(), I.data()) == B200VS_OK);
    EXPECT((int)got.size() == nq);
    for (int q = 0; q < nq && q < (int)got.size(); ++q) {
      int have = 0;
      while (have < k && I[(size_t)q * k + have] >= 0) ++have;
      EXPECT(got[q].vector_with_distances_size() == have);
      for (int i = 0; i < have && i < got[q].vector_with_distances_size(); ++i) {
        EXPECT(got[q].vector_with_distances(i).vector_with_id().id() == I[(size_t)q * k + i]);
        EXPECT(got[q].vector_with_distances(i).distance() == D[(size_t)q * k + i]);
      }
    }
  }
  void expect_range(const Results& got, const std::vector<uint8_t>& xq, int nq, float radius, int nprobe) {
    const int cap = VectorIndexB200::max_range_search_result_count;
    b200vs_search_params sp{};
    sp.nprobe = nprobe;
    std::vector<float> D((size_t)nq * cap);
    std::vector<int64_t> I((size_t)nq * cap);
    std::vector<int32_t> C(nq);
    EXPECT(b200vs_range_search_binary(h, nq, xq.data(), radius, cap, &sp, D.data(), I.data(), C.data()) == B200VS_OK);
    EXPECT((int)got.size() == nq);
    for (int q = 0; q < nq && q < (int)got.size(); ++q) {
      EXPECT(got[q].vector_with_distances_size() == C[q]);
      for (int i = 0; i < C[q] && i < got[q].vector_with_distances_size(); ++i) {
        EXPECT(got[q].vector_with_distances(i).vector_with_id().id() == I[(size_t)q * cap + i]);
        EXPECT(got[q].vector_with_distances(i).distance() == D[(size_t)q * cap + i]);
      }
    }
  }
};

// every hit: UINT8 vector of the index's dimension, metric HAMMING, distances ascending
static void expect_binary_hits(const Results& rs, int dim) {
  for (const auto& r : rs)
    for (int i = 0; i < r.vector_with_distances_size(); ++i) {
      const auto& h = r.vector_with_distances(i);
      EXPECT(h.vector_with_id().vector().value_type() == pb::common::ValueType::UINT8);
      EXPECT(h.vector_with_id().vector().dimension() == dim);
      EXPECT(h.metric_type() == pb::common::METRIC_TYPE_HAMMING);
      if (i) EXPECT(r.vector_with_distances(i - 1).distance() <= h.distance());
    }
}
static std::set<int64_t> ids_of(const Results& rs) {
  std::set<int64_t> s;
  for (const auto& r : rs)
    for (const auto& h : r.vector_with_distances()) s.insert(h.vector_with_id().id());
  return s;
}

struct EvenIds : VectorIndex::FilterFunctor {  // a functor that is neither the range nor the sort filter
  bool Check(int64_t id) override { return id % 2 == 0; }
};

static void test_create() {  // Create (test_vector_index_binary_flat.cc:71-123)
  for (auto t : {pb::common::VECTOR_INDEX_TYPE_BINARY_FLAT, pb::common::VECTOR_INDEX_TYPE_BINARY_IVF_FLAT}) {
    int64_t c = -1;
    EXPECT(make(t, pb::common::METRIC_TYPE_HAMMING, 16, 4)->GetCount(c).ok() && c == 0);
    // a binary index with another metric, or a dimension that is not whole bytes, is refused: every call then fails
    for (auto bad : {make(t, pb::common::METRIC_TYPE_L2, 16, 4), make(t, pb::common::METRIC_TYPE_NONE, 16, 4),
                     make(t, pb::common::METRIC_TYPE_HAMMING, 12, 4)}) {
      EXPECT(bad->GetCount(c).error_code() == pb::error::EINTERNAL);
      EXPECT(bad->Add(to_pb(random_rows(1, 2, 1), 1, bad->GetDimension(), 1)).error_code() == pb::error::EINTERNAL);
    }
  }
  // a float index keeps refusing UINT8 vectors
  auto fl = make(pb::common::VECTOR_INDEX_TYPE_FLAT, pb::common::METRIC_TYPE_L2, 16);
  EXPECT(fl->Add(to_pb(random_rows(2, 2, 2), 2, 16, 1)).error_code() == pb::error::EVECTOR_INVALID);
}

static void test_flat() {
  const int dim = 16, nb = 2, n = 10;  // the reference fixture: 16 bits, 10 rows
  const auto x = random_rows(n, nb, 7);
  const auto vs = to_pb(x, n, dim, 0);
  auto ix = make_ok(pb::common::VECTOR_INDEX_TYPE_BINARY_FLAT, dim);
  pb::common::VectorSearchParameter sp;
  Results results;
  // DeleteNoData, SearchNoData, RangeSearchNoData
  EXPECT(ix->Delete({}).ok());
  EXPECT(ix->Delete({1, 2, 3}).ok());
  EXPECT(ix->Search({vs[0], vs[1]}, 3, {}, false, sp, results).ok());
  EXPECT(results.size() == 2 && results[0].vector_with_distances_size() == 0);
  results.clear();
  EXPECT(ix->RangeSearch({vs[0]}, 10.1f, {}, false, sp, results).ok());
  EXPECT(results.size() == 1 && results[0].vector_with_distances_size() == 0);
  // Add: empty -> EILLEGAL_PARAMTETERS; wrong byte count, FLOAT values or a wrong dimension field -> EVECTOR_INVALID
  EXPECT(ix->Add({}).error_code() == pb::error::EILLEGAL_PARAMTETERS);
  auto bad = to_pb(x, 1, dim, 100);
  bad[0].mutable_vector()->add_binary_values(std::string(1, 'a'));
  EXPECT(ix->Add(bad).error_code() == pb::error::EVECTOR_INVALID);
  pb::common::VectorWithId fv;
  fv.set_id(100);
  fv.mutable_vector()->set_dimension(dim);
  for (int j = 0; j < dim; ++j) fv.mutable_vector()->add_float_values(0.5f);
  EXPECT(ix->Add({fv}).error_code() == pb::error::EVECTOR_INVALID);
  bad = to_pb(x, 1, dim, 100);
  bad[0].mutable_vector()->set_dimension(dim - 8);
  EXPECT(ix->Add(bad).error_code() == pb::error::EVECTOR_INVALID);
  EXPECT(ix->Search({fv}, 3, {}, false, sp, results).error_code() == pb::error::EVECTOR_INVALID);
  EXPECT(ix->Add(vs).ok());
  int64_t count = 0;
  EXPECT(ix->GetCount(count).ok() && count == n);
  // UpsertWithDuplicated
  auto dup = to_pb(x, 2, dim, 50);
  dup[1].set_id(50);
  EXPECT(ix->Upsert(dup).error_code() == pb::error::EVECTOR_ID_DUPLICATED);
  // Upsert: new rows under new ids, then new rows under existing ids
  const auto x2 = random_rows(n, nb, 8);
  EXPECT(ix->Upsert(to_pb(x2, n, dim, n)).ok());
  EXPECT(ix->GetCount(count).ok() && count == 2 * n);
  EXPECT(ix->Upsert(to_pb(x2, n, dim, n)).ok());
  EXPECT(ix->GetCount(count).ok() && count == 2 * n);
  // Search: self match at rank 0 with distance 0 (ties broken by the smaller id)
  results.clear();
  EXPECT(ix->Search({vs[3]}, 5, {}, true, sp, results).ok());  // reconstruct is ignored
  EXPECT(results.size() == 1 && results[0].vector_with_distances_size() == 5);
  EXPECT(results[0].vector_with_distances(0).distance() == 0.0f);
  EXPECT(results[0].vector_with_distances(0).vector_with_id().vector().binary_values_size() == 0);
  expect_binary_hits(results, dim);
  // filters: range + sort, sort negation, generic functor
  std::vector<int64_t> allow = {2, 4, 6, 8, 12};
  auto sortf = std::make_shared<VectorIndex::SortFilterFunctor>(allow);
  auto rangef = std::make_shared<VectorIndex::RangeFilterFunctor>(3, 9);
  results.clear();
  EXPECT(ix->Search({vs[0]}, 20, {sortf, rangef}, false, sp, results).ok());
  EXPECT((ids_of(results) == std::set<int64_t>{4, 6, 8}));
  std::vector<int64_t> deny;
  for (int64_t i = 0; i < 2 * n; i += 2) deny.push_back(i);
  auto negf = std::make_shared<VectorIndex::SortFilterFunctor>(deny, true);
  results.clear();
  EXPECT(ix->Search({vs[0], vs[1]}, 20, {negf}, false, sp, results).ok());
  for (int64_t id : ids_of(results)) EXPECT(id % 2 == 1);
  EXPECT(results.size() == 2 && results[0].vector_with_distances_size() == n);
  results.clear();
  EXPECT(ix->Search({vs[0]}, 20, {std::make_shared<EvenIds>()}, false, sp, results).ok());
  EXPECT(results.size() == 1 && results[0].vector_with_distances_size() == n);
  for (int64_t id : ids_of(results)) EXPECT(id % 2 == 0);
  results.clear();
  EXPECT(ix->RangeSearch({vs[0]}, 17.0f, {std::make_shared<EvenIds>(), rangef}, false, sp, results).ok());
  EXPECT((ids_of(results) == std::set<int64_t>{4, 6, 8}));
  // Delete, then never returned
  EXPECT(ix->Delete({3, 5}).ok());
  results.clear();
  EXPECT(ix->Search({vs[3]}, 2 * n, {}, false, sp, results).ok());
  EXPECT(results[0].vector_with_distances_size() == 2 * n - 2);
  EXPECT(!ids_of(results).count(3) && !ids_of(results).count(5));
  // RangeSearch: the radius is truncated, hits have distance < (int)radius
  results.clear();
  EXPECT(ix->RangeSearch({vs[0], vs[1]}, 6.9f, {}, false, sp, results).ok());
  for (const auto& r : results)
    for (const auto& h : r.vector_with_distances()) EXPECT(h.distance() < 6.0f);
  expect_binary_hits(results, dim);
  // the same answers as a direct call on the same rows
  Direct direct(B200VS_BINARY_FLAT, dim, 0);
  {
    std::vector<int64_t> ids(n);
    for (int i = 0; i < n; ++i) ids[i] = i;
    EXPECT(b200vs_add_with_ids_binary(direct.h, n, x.data(), ids.data(), 0) == B200VS_OK);
    for (int i = 0; i < n; ++i) ids[i] = n + i;
    EXPECT(b200vs_add_with_ids_binary(direct.h, n, x2.data(), ids.data(), 0) == B200VS_OK);
    const int64_t gone[2] = {3, 5};
    EXPECT(b200vs_remove_ids(direct.h, 2, gone, nullptr) == B200VS_OK);
  }
  const std::vector<uint8_t> xq(x.begin(), x.begin() + 4 * nb);
  const auto qs = to_pb(xq, 4, dim, 0);
  results.clear();
  EXPECT(ix->Search(qs, 7, {}, false, sp, results).ok());
  direct.expect_search(results, xq, 4, 7, 0);
  results.clear();
  EXPECT(ix->RangeSearch(qs, 6.9f, {}, false, sp, results).ok());
  direct.expect_range(results, xq, 4, 6.9f, 0);
  std::vector<float> ftrain(dim * 2);
  std::vector<uint8_t> btrain(nb * 2);
  EXPECT(ix->Train(ftrain).ok() && ix->Train(btrain).ok() && ix->Train(vs).ok());  // a Flat index needs no training
  EXPECT(!ix->NeedTrain() && ix->IsTrained() && !ix->SupportSave() && !ix->IsExceedsMaxElements(1 << 30));
}

static void test_flat_large() {  // marshalling of wider rows and more queries than the coalescer's batch limit
  const int dim = 256, nb = 32, n = 3000, nq = 100, k = 10;
  const auto x = random_rows(n, nb, 9);
  auto ix = make_ok(pb::common::VECTOR_INDEX_TYPE_BINARY_FLAT, dim);
  EXPECT(ix->Add(to_pb(x, n, dim, 1000)).ok());
  Direct direct(B200VS_BINARY_FLAT, dim, 0);
  std::vector<int64_t> ids(n);
  for (int i = 0; i < n; ++i) ids[i] = 1000 + i;
  EXPECT(b200vs_add_with_ids_binary(direct.h, n, x.data(), ids.data(), 0) == B200VS_OK);
  const auto xq = random_rows(nq, nb, 10);
  Results results;
  EXPECT(ix->Search(to_pb(xq, nq, dim, 0), k, {}, false, pb::common::VectorSearchParameter(), results).ok());
  direct.expect_search(results, xq, nq, k, 0);
  expect_binary_hits(results, dim);
  results.clear();
  EXPECT(ix->RangeSearch(to_pb(xq, 5, dim, 0), 110.0f, {}, false, pb::common::VectorSearchParameter(), results).ok());
  direct.expect_range(results, std::vector<uint8_t>(xq.begin(), xq.begin() + 5 * nb), 5, 110.0f, 0);
}

static void test_ivf() {
  const int dim = 64, nb = 8, n = 2000, nlist = 8, nq = 6, k = 10;
  const auto x = random_rows(n, nb, 11);
  const auto vs = to_pb(x, n, dim, 0);
  const std::vector<uint8_t> xq(x.begin(), x.begin() + nq * nb);
  const auto qs = to_pb(xq, nq, dim, 0);
  pb::common::VectorSearchParameter sp;
  Results results;
  auto ix = make_ok(pb::common::VECTOR_INDEX_TYPE_BINARY_IVF_FLAT, dim, nlist);
  EXPECT(ix->NeedTrain() && !ix->IsTrained() && !ix->IsExceedsMaxElements(1 << 30));
  // SearchNotTrain / RangeSearch / Delete before training
  EXPECT(ix->Search(qs, k, {}, false, sp, results).ok());
  EXPECT((int)results.size() == nq && results[0].vector_with_distances_size() == 0);
  results.clear();
  EXPECT(ix->RangeSearch(qs, 30.0f, {}, false, sp, results).ok());
  EXPECT((int)results.size() == nq && results[0].vector_with_distances_size() == 0);
  EXPECT(ix->Delete({1, 2}).ok());
  // Train(float) is an error, not an abort; bad byte counts are refused
  std::vector<float> ftrain(dim * 100, 0.5f);
  EXPECT(ix->Train(ftrain).error_code() == pb::error::EILLEGAL_PARAMTETERS);
  std::vector<uint8_t> none, ragged(nb * 10 + 3);
  EXPECT(ix->Train(none).error_code() == pb::error::EILLEGAL_PARAMTETERS);
  EXPECT(ix->Train(ragged).error_code() == pb::error::EILLEGAL_PARAMTETERS);
  EXPECT(!ix->IsTrained());
  // AddNotTrain: Add trains with its own batch, then adds
  EXPECT(ix->Add(vs).ok());
  EXPECT(ix->IsTrained());
  int64_t count = 0;
  EXPECT(ix->GetCount(count).ok() && count == n);
  // the same rows through the C ABI: the same training rows give the same centroids (training is deterministic)
  Direct direct(B200VS_BINARY_IVF_FLAT, dim, nlist);
  std::vector<int64_t> ids(n);
  for (int i = 0; i < n; ++i) ids[i] = i;
  EXPECT(b200vs_train_binary(direct.h, n, x.data()) == B200VS_OK);
  EXPECT(b200vs_add_with_ids_binary(direct.h, n, x.data(), ids.data(), 0) == B200VS_OK);
  for (int nprobe : {0, 1, 3}) {
    sp.mutable_binary_ivf_flat()->set_nprobe(nprobe);
    results.clear();
    EXPECT(ix->Search(qs, k, {}, false, sp, results).ok());
    direct.expect_search(results, xq, nq, k, nprobe);
    expect_binary_hits(results, dim);
    EXPECT(results[0].vector_with_distances(0).vector_with_id().id() == 0 && results[0].vector_with_distances(0).distance() == 0.0f);
    results.clear();
    EXPECT(ix->RangeSearch(qs, 25.5f, {}, false, sp, results).ok());
    direct.expect_range(results, xq, nq, 25.5f, nprobe);
  }
  // the nprobe knob: nprobe = nlist probes every list, so the results are the Flat results
  auto flat = make_ok(pb::common::VECTOR_INDEX_TYPE_BINARY_FLAT, dim);
  EXPECT(flat->Add(vs).ok());
  Results want;
  EXPECT(flat->Search(qs, k, {}, false, sp, want).ok());
  sp.mutable_binary_ivf_flat()->set_nprobe(nlist);
  results.clear();
  EXPECT(ix->Search(qs, k, {}, false, sp, results).ok());
  EXPECT(results.size() == want.size());
  for (size_t q = 0; q < results.size() && q < want.size(); ++q) {
    EXPECT(results[q].vector_with_distances_size() == want[q].vector_with_distances_size());
    for (int i = 0; i < results[q].vector_with_distances_size() && i < want[q].vector_with_distances_size(); ++i) {
      EXPECT(results[q].vector_with_distances(i).vector_with_id().id() == want[q].vector_with_distances(i).vector_with_id().id());
      EXPECT(results[q].vector_with_distances(i).distance() == want[q].vector_with_distances(i).distance());
    }
  }
  // filters on a trained IVF index
  std::vector<int64_t> allow;
  for (int64_t i = 0; i < n; i += 3) allow.push_back(i);
  const std::set<int64_t> allowed(allow.begin(), allow.end());
  results.clear();
  EXPECT(ix->Search(qs, k, {std::make_shared<VectorIndex::SortFilterFunctor>(allow)}, false, sp, results).ok());
  for (int64_t id : ids_of(results)) EXPECT(allowed.count(id) == 1);
  results.clear();
  EXPECT(ix->Search(qs, k, {std::make_shared<EvenIds>()}, false, sp, results).ok());
  for (int64_t id : ids_of(results)) EXPECT(id % 2 == 0);
  // Delete: unknown ids -> EVECTOR_INVALID (ivf_flat.cc:180-184); known ids are gone
  EXPECT(ix->Delete({123456}).error_code() == pb::error::EVECTOR_INVALID);
  EXPECT(ix->Delete({0}).ok());
  results.clear();
  EXPECT(ix->Search({qs[0]}, k, {}, false, sp, results).ok());
  EXPECT(!ids_of(results).count(0));
  // Train from uint8_t rows and from VectorWithId: the same centroids as the auto-train, so the same answers
  std::vector<uint8_t> btrain(x);
  auto ix2 = make_ok(pb::common::VECTOR_INDEX_TYPE_BINARY_IVF_FLAT, dim, nlist);
  EXPECT(ix2->Train(btrain).ok() && ix2->IsTrained());
  auto ix3 = make_ok(pb::common::VECTOR_INDEX_TYPE_BINARY_IVF_FLAT, dim, nlist);
  EXPECT(ix3->Train(vs).ok() && ix3->IsTrained());
  sp.mutable_binary_ivf_flat()->set_nprobe(2);
  for (auto* t : {ix2.get(), ix3.get()}) {
    EXPECT(t->Add(vs).ok());
    results.clear();
    EXPECT(t->Search(qs, k, {}, false, sp, results).ok());
    direct.expect_search(results, xq, nq, k, 2);
  }
  auto ix4 = make_ok(pb::common::VECTOR_INDEX_TYPE_BINARY_IVF_FLAT, dim, nlist);
  auto short_row = to_pb(x, 3, dim, 0);
  short_row[1].mutable_vector()->mutable_binary_values()->pop_back();
  EXPECT(ix4->Train(short_row).error_code() == pb::error::EINTERNAL);
  EXPECT(!ix4->IsTrained());
  // Save -> Load: identical search and range-search results
  const std::string path = std::string(getenv("TMPDIR") ? getenv("TMPDIR") : "/tmp") + "/test_plugin_binary_" + std::to_string(getpid()) + ".idx";
  EXPECT(ix2->Save(path).ok());
  auto loaded = make_ok(pb::common::VECTOR_INDEX_TYPE_BINARY_IVF_FLAT, dim, nlist);
  EXPECT(loaded->Load(path).ok() && loaded->IsTrained());
  EXPECT(loaded->GetCount(count).ok() && count == n);
  Results a, b;
  EXPECT(ix2->Search(qs, k, {}, false, sp, a).ok() && loaded->Search(qs, k, {}, false, sp, b).ok());
  EXPECT(a.size() == b.size());
  for (size_t q = 0; q < a.size() && q < b.size(); ++q) {
    EXPECT(a[q].vector_with_distances_size() == b[q].vector_with_distances_size());
    for (int i = 0; i < a[q].vector_with_distances_size() && i < b[q].vector_with_distances_size(); ++i)
      EXPECT(a[q].vector_with_distances(i).vector_with_id().id() == b[q].vector_with_distances(i).vector_with_id().id() &&
             a[q].vector_with_distances(i).distance() == b[q].vector_with_distances(i).distance());
  }
  results.clear();
  EXPECT(loaded->RangeSearch(qs, 25.5f, {}, false, sp, results).ok());
  direct.expect_range(results, xq, nq, 25.5f, 2);
  unlink(path.c_str());
}

static void test_calc_distance() {  // CalcDistanceEntry with METRIC_TYPE_HAMMING (vector_index_utils.cc:146-149, :333-357)
  auto vec = [](std::initializer_list<int> bytes) {
    pb::common::Vector v;
    for (int b : bytes) v.add_binary_values(std::string(1, (char)b));
    return v;
  };
  std::vector<pb::common::Vector> left{vec({0x0F, 0x00}), vec({0xFF, 0xFF})}, right{vec({0xFF, 0x00}), vec({0x0F, 0x00}), vec({0x00, 0x81})}, rl, rr;
  std::vector<std::vector<float>> dist;
  EXPECT(VectorIndexB200Utils::CalcDistance(1, pb::common::METRIC_TYPE_HAMMING, left, right, false, dist, rl, rr).ok());
  EXPECT((dist == std::vector<std::vector<float>>{{4, 0, 6}, {8, 12, 14}}));
  EXPECT(rl.empty() && rr.empty());
  EXPECT(VectorIndexB200Utils::CalcDistance(1, pb::common::METRIC_TYPE_HAMMING, left, right, true, dist, rl, rr).ok());
  EXPECT(rl.size() == 2 && rr.size() == 3);
  for (size_t i = 0; i < rl.size(); ++i)
    EXPECT(rl[i].binary_values() == left[i].binary_values() && rl[i].dimension() == 16 && rl[i].value_type() == pb::common::ValueType::UINT8);
  for (size_t i = 0; i < rr.size(); ++i)
    EXPECT(rr[i].binary_values() == right[i].binary_values() && rr[i].dimension() == 16 && rr[i].value_type() == pb::common::ValueType::UINT8);
  // a vector of another byte count is refused
  std::vector<pb::common::Vector> ragged{vec({0x01, 0x02, 0x03})};
  EXPECT(VectorIndexB200Utils::CalcDistance(1, pb::common::METRIC_TYPE_HAMMING, left, ragged, false, dist, rl, rr).error_code() == pb::error::EILLEGAL_PARAMTETERS);
  EXPECT(VectorIndexB200Utils::CalcDistance(1, pb::common::METRIC_TYPE_HAMMING, ragged, right, false, dist, rl, rr).error_code() == pb::error::EILLEGAL_PARAMTETERS);
  // empty operands: one empty row per left vector
  EXPECT(VectorIndexB200Utils::CalcDistance(1, pb::common::METRIC_TYPE_HAMMING, left, {}, false, dist, rl, rr).ok());
  EXPECT(dist.size() == 2 && dist[0].empty());
  // HNSWLIB has no HAMMING case: OK, and nothing is touched
  std::vector<std::vector<float>> keep{{7.0f}};
  std::vector<pb::common::Vector> kl{vec({1})}, kr;
  EXPECT(VectorIndexB200Utils::CalcDistance(2, pb::common::METRIC_TYPE_HAMMING, left, right, true, keep, kl, kr).ok());
  EXPECT((keep == std::vector<std::vector<float>>{{7.0f}}) && kl.size() == 1 && kr.empty());
}

int main() {
  test_create();
  test_flat();
  test_flat_large();
  test_ivf();
  test_calc_distance();
  printf(g_fail ? "PLUGIN BINARY TESTS FAILED: %d\n" : "PLUGIN BINARY TESTS OK%.0d\n", g_fail);
  return g_fail ? 1 : 0;
}
