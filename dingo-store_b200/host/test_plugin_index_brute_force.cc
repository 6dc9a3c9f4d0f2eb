// test_plugin_index_brute_force.cc — VectorIndexB200::BruteForceSearch / BruteForceRangeSearch, the reader's brute-force
// loops answered from the region's own index.  Each index goes through adds, deletes and upserts; its live rows inside the
// region's range [min, max) are kept on the host in ascending id order and replayed, as the reader's RocksDB loop does, in
// 2048-row batches through BruteForceScannerB200 / BruteForceRangeScannerB200.  The plugin methods must return the same
// results hit by hit (ids, distance bits, metric, dimension), with the filters lowered as Search lowers them; the top-k
// scanner takes no filters, so it is fed only the rows that pass them.  The types the library does not serve come back
// as EVECTOR_NOT_SUPPORT.  Needs a GPU; run by tests/test_gpu_plugin_index_brute_force.py.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <random>
#include <vector>

#include "vector_index_b200.h"

using namespace dingodb;
using Results = std::vector<pb::index::VectorWithDistanceResult>;
using Filters = std::vector<std::shared_ptr<VectorIndex::FilterFunctor>>;

static int g_fail = 0;
#define EXPECT(cond)                                                                \
  do {                                                                              \
    if (!(cond)) { ++g_fail; printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); } \
  } while (0)

constexpr int kBatch = 2048;  // FLAGS_vector_index_bruteforce_batch_count
constexpr int kDim = 64;
constexpr int64_t kMin = 1000, kMax = 9000;  // the region's ids

class FnFilter : public VectorIndex::FilterFunctor {
 public:
  explicit FnFilter(std::function<bool(int64_t)> f) : f_(std::move(f)) {}
  bool Check(int64_t id) override { return f_(id); }
 private:
  std::function<bool(int64_t)> f_;
};

// IP rows on a grid (integers in [-4, 4] * 2^-6): every ip and 1 - ip is exact, so no two rows share a distance without
// sharing an ip, and any batching of the scan gives the same top-k
static std::vector<float> rows(int n, unsigned seed, bool grid) {
  std::mt19937 rng(seed);
  std::normal_distribution<float> nd;
  std::uniform_int_distribution<int> ui(-4, 4);
  std::vector<float> x((size_t)n * kDim);
  for (auto& v : x) v = grid ? (float)ui(rng) / 64.f : nd(rng);
  return x;
}
static std::vector<pb::common::VectorWithId> to_pb(const std::vector<float>& x, const std::vector<int64_t>& ids) {
  std::vector<pb::common::VectorWithId> out(ids.size());
  for (size_t i = 0; i < ids.size(); ++i) {
    out[i].set_id(ids[i]);
    out[i].mutable_vector()->set_dimension(kDim);
    out[i].mutable_vector()->set_value_type(pb::common::ValueType::FLOAT);
    out[i].mutable_vector()->mutable_float_values()->assign(x.begin() + i * kDim, x.begin() + (i + 1) * kDim);
  }
  return out;
}
static std::shared_ptr<VectorIndexB200> make(pb::common::VectorIndexType type, pb::common::MetricType m) {
  pb::common::VectorIndexParameter p;
  p.set_vector_index_type(type);
  if (type == pb::common::VECTOR_INDEX_TYPE_IVF_FLAT) {
    auto* q = p.mutable_ivf_flat_parameter();
    q->dimension_ = kDim; q->metric_type_ = m; q->ncentroids_ = 16;
  } else if (type == pb::common::VECTOR_INDEX_TYPE_IVF_PQ) {
    auto* q = p.mutable_ivf_pq_parameter();
    q->dimension_ = kDim; q->metric_type_ = m; q->ncentroids_ = 4; q->nsubvector_ = 8; q->nbits_per_idx_ = 4;
  } else if (type == pb::common::VECTOR_INDEX_TYPE_HNSW) {
    auto* q = p.mutable_hnsw_parameter();
    q->dimension_ = kDim; q->metric_type_ = m; q->nlinks_ = 16; q->efconstruction_ = 64; q->max_elements_ = 40000;
  } else if (type == pb::common::VECTOR_INDEX_TYPE_BINARY_FLAT) {
    auto* q = p.mutable_binary_flat_parameter();
    q->dimension_ = kDim; q->metric_type_ = m;
  } else {
    auto* q = p.mutable_flat_parameter();
    q->dimension_ = kDim; q->metric_type_ = m;
  }
  return std::make_shared<VectorIndexB200>(1, p, pb::common::RegionEpoch(), pb::common::Range(), nullptr);
}

using Model = std::map<int64_t, std::vector<float>>;  // the live rows by id

// adds (ids 0..11999 shuffled, so the index also holds rows outside the region), deletes and upserts, mirrored in m
static void fill(VectorIndexB200& ix, Model& m, bool grid, bool trained) {
  const int n = 12000;
  std::vector<int64_t> ids(n);
  for (int i = 0; i < n; ++i) ids[i] = i;
  std::shuffle(ids.begin(), ids.end(), std::mt19937(11));
  std::vector<float> x = rows(n, 12, grid);
  if (trained) { std::vector<float> t(x.begin(), x.begin() + 4096 * kDim); EXPECT(ix.Train(t).ok()); }
  EXPECT(ix.Add(to_pb(x, ids)).ok());
  for (int i = 0; i < n; ++i) m[ids[i]].assign(x.begin() + (size_t)i * kDim, x.begin() + (size_t)(i + 1) * kDim);
  std::vector<int64_t> dead;
  for (int i = 0; i < n; i += 3) dead.push_back(ids[i]);
  EXPECT(ix.Delete(dead).ok());
  for (int64_t id : dead) m.erase(id);
  std::vector<int64_t> up;
  for (int i = 1; i < n; i += 7) up.push_back(ids[i]);
  std::vector<float> xu = rows((int)up.size(), 13, grid);
  EXPECT(ix.Upsert(to_pb(xu, up)).ok());
  for (size_t i = 0; i < up.size(); ++i) m[up[i]].assign(xu.begin() + i * kDim, xu.begin() + (i + 1) * kDim);
}

// the region's live rows that pass `pass`, in ascending id order (RocksDB key order)
static std::vector<pb::common::VectorWithId> region_rows(const Model& m, const std::function<bool(int64_t)>& pass) {
  std::vector<int64_t> ids;
  std::vector<float> x;
  for (const auto& kv : m)
    if (kv.first >= kMin && kv.first < kMax && pass(kv.first)) { ids.push_back(kv.first); x.insert(x.end(), kv.second.begin(), kv.second.end()); }
  return to_pb(x, ids);
}

template <class Scanner>
static void replay(Scanner& sc, const std::vector<pb::common::VectorWithId>& rs, Results& out) {
  for (size_t a = 0; a < rs.size(); a += kBatch) {
    std::vector<pb::common::VectorWithId> batch(rs.begin() + a, rs.begin() + std::min(rs.size(), a + kBatch));
    EXPECT(sc.Push(batch).ok());
  }
  EXPECT(sc.Finish(out).ok());
}

static bool same_bits(float a, float b) { return memcmp(&a, &b, 4) == 0; }

static int64_t expect_same(const Results& got, const Results& want, const char* what) {
  EXPECT(got.size() == want.size());
  int bad = 0;
  int64_t hits = 0;
  for (size_t q = 0; q < got.size() && q < want.size(); ++q) {
    if (got[q].vector_with_distances_size() != want[q].vector_with_distances_size()) { ++bad; continue; }
    for (int i = 0; i < want[q].vector_with_distances_size(); ++i) {
      const auto& a = got[q].vector_with_distances(i);
      const auto& b = want[q].vector_with_distances(i);
      if (a.vector_with_id().id() != b.vector_with_id().id() || !same_bits(a.distance(), b.distance()) || a.metric_type() != b.metric_type() ||
          a.vector_with_id().vector().dimension() != b.vector_with_id().vector().dimension() ||
          a.vector_with_id().vector().value_type() != b.vector_with_id().vector().value_type())
        ++bad;
      ++hits;
    }
  }
  if (bad) printf("  %s: %d mismatching queries / hits\n", what, bad);
  EXPECT(bad == 0);
  return hits;
}

static void check(const char* name, pb::common::VectorIndexType type, pb::common::MetricType metric, bool grid) {
  auto ix = make(type, metric);
  Model m;
  fill(*ix, m, grid, type == pb::common::VECTOR_INDEX_TYPE_IVF_FLAT);
  const auto queries = to_pb(rows(6, 14, grid), std::vector<int64_t>(6, 0));
  std::vector<int64_t> deny;
  for (int64_t id = kMin; id < kMax; id += 4) deny.push_back(id);
  auto generic = [](int64_t id) { return id % 5 != 0; };
  auto not_denied = [deny](int64_t id) { return !std::binary_search(deny.begin(), deny.end(), id); };
  auto in_range = [](int64_t id) { return id >= 2000 && id < 20000; };
  struct Case { const char* name; bool g, s, r; };
  for (const Case c : {Case{"region only", false, false, false}, Case{"generic", true, false, false},
                       Case{"negated sort", false, true, false}, Case{"range over the region edge", false, false, true},
                       Case{"all three", true, true, true}}) {
    auto filters = [&]() {
      Filters fs;
      if (c.g) fs.push_back(std::make_shared<FnFilter>(generic));
      if (c.s) { std::vector<int64_t> l = deny; fs.push_back(std::make_shared<VectorIndex::SortFilterFunctor>(l, true)); }
      if (c.r) fs.push_back(std::make_shared<VectorIndex::RangeFilterFunctor>(2000, 20000));
      return fs;
    };
    auto pass = [&](int64_t id) { return (!c.g || generic(id)) && (!c.s || not_denied(id)) && (!c.r || in_range(id)); };
    for (uint32_t topk : {1u, 100u, 5000u}) {
      Results got, want;
      EXPECT(ix->BruteForceSearch(queries, topk, kMin, kMax, filters(), got).ok());
      BruteForceScannerB200 sc(metric, kDim, queries, topk);
      replay(sc, region_rows(m, pass), want);
      EXPECT(expect_same(got, want, name) > 0);
    }
    {
      const float radius = metric == pb::common::METRIC_TYPE_L2 ? 100.f : 0.98f;  // a few percent of the rows
      Results got, want;
      EXPECT(ix->BruteForceRangeSearch(queries, radius, kMin, kMax, filters(), got).ok());
      BruteForceRangeScannerB200 sc(metric, kDim, queries, radius, filters());
      replay(sc, region_rows(m, [](int64_t) { return true; }), want);
      EXPECT(expect_same(got, want, name) > 0);
    }
  }
  printf("  %s ok\n", name);
}

static void refusals() {
  const auto queries = to_pb(rows(2, 15, false), {0, 0});
  std::vector<float> x = rows(5000, 16, false);
  std::vector<int64_t> ids(5000);
  for (int i = 0; i < 5000; ++i) ids[i] = i;
  auto pq = make(pb::common::VECTOR_INDEX_TYPE_IVF_PQ, pb::common::METRIC_TYPE_L2);
  EXPECT(pq->Train(x).ok());
  auto hc = make(pb::common::VECTOR_INDEX_TYPE_HNSW, pb::common::METRIC_TYPE_COSINE);
  auto bf = make(pb::common::VECTOR_INDEX_TYPE_BINARY_FLAT, pb::common::METRIC_TYPE_HAMMING);
  for (auto& ix : {pq, hc, bf}) {
    if (ix != bf) EXPECT(ix->Add(to_pb(x, ids)).ok());
    Results r;
    auto st = ix->BruteForceSearch(queries, 10, 0, 5000, {}, r);
    EXPECT(!st.ok() && st.error_code() == pb::error::EVECTOR_NOT_SUPPORT);
    st = ix->BruteForceRangeSearch(queries, 1.0f, 0, 5000, {}, r);
    EXPECT(!st.ok() && st.error_code() == pb::error::EVECTOR_NOT_SUPPORT);
  }
  auto fl = make(pb::common::VECTOR_INDEX_TYPE_FLAT, pb::common::METRIC_TYPE_L2);
  Results r;
  auto st = fl->BruteForceSearch({}, 10, 0, 10, {}, r);
  EXPECT(!st.ok() && st.error_code() == pb::error::EILLEGAL_PARAMTETERS);
  EXPECT(fl->BruteForceSearch(queries, 10, 0, 10, {}, r).ok());  // an empty index: one empty result per query
  EXPECT(r.size() == 2 && r[0].vector_with_distances_size() == 0);
}

int main() {
  {
    b200vs_index* h = nullptr;
    if (b200vs_create(B200VS_FLAT, B200VS_L2, 8, nullptr, &h) != B200VS_OK) {
      printf("cannot create an index: %s\n", b200vs_last_error());  // no CUDA device: the product has no CPU fallback
      return 2;
    }
    b200vs_destroy(h);
  }
  check("flat l2", pb::common::VECTOR_INDEX_TYPE_FLAT, pb::common::METRIC_TYPE_L2, false);
  check("ivf_flat ip", pb::common::VECTOR_INDEX_TYPE_IVF_FLAT, pb::common::METRIC_TYPE_INNER_PRODUCT, true);
  check("hnsw l2", pb::common::VECTOR_INDEX_TYPE_HNSW, pb::common::METRIC_TYPE_L2, false);
  refusals();
  if (g_fail) { printf("%d FAILURES\n", g_fail); return 1; }
  printf("PLUGIN INDEX BRUTE FORCE TESTS OK\n");
  return 0;
}
