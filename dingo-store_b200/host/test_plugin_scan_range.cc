// test_plugin_scan_range.cc — BruteForceRangeScannerB200, the GPU form of the loop of VectorReader::BruteForceRangeSearch
// (src/vector/vector_reader.cc:2050-2202).  The reader's loop is replayed in 2048-row batches and every result is
// compared with a restatement of the rule: per query, the first max_range_search_result_count hits in scan order, a hit
// being a row whose FP32 value (quad_distance's summation order, restated below) is strictly inside the radius and which
// every filter passes; ids and distance bits must match.  Cosine, whose normalisation is not restated here, is compared
// with a Flat VectorIndexB200's RangeSearch over the same rows instead.  Needs a GPU; run by
// tests/test_gpu_plugin_scan_range.py.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <random>
#include <string>

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

// A functor the GPU form has no device counterpart for: applied on the host by Push.
class FnFilter : public VectorIndex::FilterFunctor {
 public:
  explicit FnFilter(std::function<bool(int64_t)> f) : f_(std::move(f)) {}
  bool Check(int64_t id) override { return f_(id); }
 private:
  std::function<bool(int64_t)> f_;
};

static std::vector<float> random_rows(int n, int d, unsigned seed) {
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> u(0.f, 1.f);
  std::vector<float> x((size_t)n * d);
  for (auto& v : x) v = u(rng);
  return x;
}
static std::vector<pb::common::VectorWithId> to_pb(const std::vector<float>& x, const std::vector<int64_t>& ids, int d) {
  std::vector<pb::common::VectorWithId> out(ids.size());
  for (size_t i = 0; i < ids.size(); ++i) {
    out[i].set_id(ids[i]);
    auto* v = out[i].mutable_vector();
    v->set_dimension(d);
    v->set_value_type(pb::common::ValueType::FLOAT);
    v->mutable_float_values()->assign(x.begin() + i * d, x.begin() + (i + 1) * d);
  }
  return out;
}

// The exact scan's per-row value in quad_distance's order (csrc/common.cuh): 16 lane partials, fold 16 -> 8, 8-wide tail,
// fold 8 -> 4, 4-wide tail, zero-filled 1..3 tail, (m0 + m1) + (m2 + m3).  L2: squared distance; IP: inner product.
static float raw_value(const float* x, const float* q, int d, bool l2) {
  auto term = [&](int i) { if (l2) { const float t = x[i] - q[i]; return t * t; } return x[i] * q[i]; };
  float acc[16] = {0};
  const int nfull = d / 16;
  for (int c = 0; c < nfull; ++c)
    for (int j = 0; j < 16; ++j) acc[j] = acc[j] + term(16 * c + j);
  float m1[8], m2[4];
  for (int j = 0; j < 8; ++j) m1[j] = acc[8 + j] + acc[j];
  int base = 16 * nfull, rem = d - base;
  if (rem >= 8) { for (int j = 0; j < 8; ++j) m1[j] = m1[j] + term(base + j); base += 8; rem -= 8; }
  for (int j = 0; j < 4; ++j) m2[j] = m1[4 + j] + m1[j];
  if (rem >= 4) { for (int j = 0; j < 4; ++j) m2[j] = m2[j] + term(base + j); base += 4; rem -= 4; }
  if (rem > 0) for (int j = 0; j < 4; ++j) m2[j] = m2[j] + (j < rem ? term(base + j) : 0.f);
  return (m2[0] + m2[1]) + (m2[2] + m2[3]);
}

struct Hit { int64_t id; float dist; };

// The rule: rows in scan order, L2 dist < radius or IP ip > 1 - radius, every filter passes, at most cap hits per query.
static std::vector<std::vector<Hit>> restated(const std::vector<float>& xq, int nq, const std::vector<float>& xb,
                                              const std::vector<int64_t>& ids, int d, bool l2, float radius, int cap,
                                              const std::function<bool(int64_t)>& pass) {
  std::vector<std::vector<Hit>> out(nq);
  const float thr = l2 ? radius : 1.0f - radius;
  for (int q = 0; q < nq; ++q)
    for (size_t r = 0; r < ids.size() && (int)out[q].size() < cap; ++r) {
      if (ids[r] < 0 || !pass(ids[r])) continue;
      const float v = raw_value(xb.data() + r * d, xq.data() + (size_t)q * d, d, l2);
      if (l2 ? v < thr : v > thr) out[q].push_back({ids[r], l2 ? v : 1.0f - v});
    }
  return out;
}

static bool same_bits(float a, float b) { return memcmp(&a, &b, 4) == 0; }

static void expect_equal(const Results& got, const std::vector<std::vector<Hit>>& want, int d, pb::common::MetricType m, const char* what) {
  EXPECT(got.size() == want.size());
  int bad = 0;
  for (size_t q = 0; q < got.size() && q < want.size(); ++q) {
    if (got[q].vector_with_distances_size() != (int)want[q].size()) { ++bad; continue; }
    for (size_t i = 0; i < want[q].size(); ++i) {
      const auto& h = got[q].vector_with_distances((int)i);
      if (h.vector_with_id().id() != want[q][i].id || !same_bits(h.distance(), want[q][i].dist) || h.metric_type() != m ||
          h.vector_with_id().vector().dimension() != d || h.vector_with_id().vector().value_type() != pb::common::ValueType::FLOAT)
        ++bad;
    }
  }
  if (bad) printf("  %s: %d mismatching queries / hits\n", what, bad);
  EXPECT(bad == 0);
}

// The reader's loop: push every full batch, then the remainder, then collect.
static butil::Status replay(BruteForceRangeScannerB200& sc, const std::vector<pb::common::VectorWithId>& rows, Results& out) {
  for (size_t a = 0; a < rows.size(); a += kBatch) {
    std::vector<pb::common::VectorWithId> batch(rows.begin() + a, rows.begin() + std::min(rows.size(), a + kBatch));
    auto st = sc.Push(batch);
    if (!st.ok()) return st;
  }
  return sc.Finish(out);
}

// the radius that keeps about `frac` of the rows for query 0
static float radius_for(const std::vector<float>& xq, const std::vector<float>& xb, int n, int d, bool l2, double frac) {
  std::vector<float> v(n);
  for (int r = 0; r < n; ++r) v[r] = raw_value(xb.data() + (size_t)r * d, xq.data(), d, l2);
  std::sort(v.begin(), v.end());
  const float t = l2 ? v[(size_t)(frac * n)] : v[n - 1 - (size_t)(frac * n)];
  return l2 ? t : 1.0f - t;
}

static void test_filters_l2() {
  const int d = 96, n = 5000, nq = 4;
  std::vector<float> xb = random_rows(n, d, 1), xq = random_rows(nq, d, 2);
  std::vector<int64_t> ids(n);
  for (int i = 0; i < n; ++i) ids[i] = i + 1;
  std::shuffle(ids.begin(), ids.end(), std::mt19937(3));
  const auto rows = to_pb(xb, ids, d);
  const auto queries = to_pb(xq, std::vector<int64_t>(nq, 0), d);
  const float radius = radius_for(xq, xb, n, d, true, 0.05);
  std::vector<int64_t> deny;
  for (int i = 0; i < n; i += 5) deny.push_back(ids[i]);
  std::sort(deny.begin(), deny.end());
  auto generic = [](int64_t id) { return id % 3 != 0; };
  auto in_range = [](int64_t id) { return id >= 100 && id < 4000; };
  auto not_denied = [deny](int64_t id) { return !std::binary_search(deny.begin(), deny.end(), id); };
  struct Case { const char* name; bool g, r, s; };
  for (const Case c : {Case{"no filter", false, false, false}, Case{"generic", true, false, false}, Case{"range", false, true, false},
                       Case{"negated sort", false, false, true}, Case{"all three", true, true, true}}) {
    Filters fs;
    if (c.g) fs.push_back(std::make_shared<FnFilter>(generic));
    if (c.r) fs.push_back(std::make_shared<VectorIndex::RangeFilterFunctor>(100, 4000));
    if (c.s) { std::vector<int64_t> l = deny; fs.push_back(std::make_shared<VectorIndex::SortFilterFunctor>(l, true)); }
    BruteForceRangeScannerB200 sc(pb::common::METRIC_TYPE_L2, d, queries, radius, fs);
    Results got;
    EXPECT(replay(sc, rows, got).ok());
    auto pass = [&](int64_t id) { return (!c.g || generic(id)) && (!c.r || in_range(id)) && (!c.s || not_denied(id)); };
    const auto want = restated(xq, nq, xb, ids, d, true, radius, VectorIndexB200::max_range_search_result_count, pass);
    EXPECT(!want[0].empty());
    expect_equal(got, want, d, pb::common::METRIC_TYPE_L2, c.name);
  }
}

static void test_cap_ip() {  // the cap is reached inside the first batch; later hits are dropped, nothing is sorted
  const int d = 13, n = 6000, nq = 3;
  std::vector<float> xb = random_rows(n, d, 4), xq = random_rows(nq, d, 5);
  std::vector<int64_t> ids(n);
  for (int i = 0; i < n; ++i) ids[i] = 10 * i + 7;
  const auto rows = to_pb(xb, ids, d);
  const auto queries = to_pb(xq, std::vector<int64_t>(nq, 0), d);
  const float radius = radius_for(xq, xb, n, d, false, 0.3);
  const int32_t saved = VectorIndexB200::max_range_search_result_count;
  VectorIndexB200::max_range_search_result_count = 50;
  BruteForceRangeScannerB200 sc(pb::common::METRIC_TYPE_INNER_PRODUCT, d, queries, radius, {});
  VectorIndexB200::max_range_search_result_count = saved;
  Results got;
  EXPECT(replay(sc, rows, got).ok());
  const auto want = restated(xq, nq, xb, ids, d, false, radius, 50, [](int64_t) { return true; });
  EXPECT(want[0].size() == 50);
  expect_equal(got, want, d, pb::common::METRIC_TYPE_INNER_PRODUCT, "ip cap 50");
}

static void test_cosine_matches_flat_range_search() {
  const int d = 64, n = 4500, nq = 5;
  std::vector<float> xb = random_rows(n, d, 6), xq = random_rows(nq, d, 7);
  std::vector<int64_t> ids(n);
  for (int i = 0; i < n; ++i) ids[i] = i + 1000;
  const auto rows = to_pb(xb, ids, d);
  const auto queries = to_pb(xq, std::vector<int64_t>(nq, 0), d);
  const float radius = 0.2f;
  const int32_t saved = VectorIndexB200::max_range_search_result_count;
  VectorIndexB200::max_range_search_result_count = n + 1;  // no cap: the Flat search keeps the closest hits, the scan the first
  BruteForceRangeScannerB200 sc(pb::common::METRIC_TYPE_COSINE, d, queries, radius, {});
  Results got;
  EXPECT(replay(sc, rows, got).ok());
  pb::common::VectorIndexParameter p;
  p.set_vector_index_type(pb::common::VECTOR_INDEX_TYPE_FLAT);
  p.mutable_flat_parameter()->dimension_ = d;
  p.mutable_flat_parameter()->metric_type_ = pb::common::METRIC_TYPE_COSINE;
  VectorIndexB200 flat(1, p, pb::common::RegionEpoch(), pb::common::Range(), nullptr);
  EXPECT(flat.Add(rows).ok());
  Results want;
  EXPECT(flat.RangeSearch(queries, radius, {}, false, pb::common::VectorSearchParameter(), want).ok());
  VectorIndexB200::max_range_search_result_count = saved;
  EXPECT(got.size() == want.size());
  int total = 0;
  for (size_t q = 0; q < got.size() && q < want.size(); ++q) {  // same (id, distance bits) set; the scan keeps scan order
    std::map<int64_t, float> a, b;
    for (const auto& h : got[q].vector_with_distances()) a[h.vector_with_id().id()] = h.distance();
    for (const auto& h : want[q].vector_with_distances()) b[h.vector_with_id().id()] = h.distance();
    EXPECT(a.size() == b.size() && (int)a.size() <= n);
    for (const auto& kv : a) EXPECT(b.count(kv.first) && same_bits(b[kv.first], kv.second));
    int64_t prev = -1;
    for (const auto& h : got[q].vector_with_distances()) { EXPECT(h.vector_with_id().id() > prev); prev = h.vector_with_id().id(); }
    total += (int)a.size();
  }
  EXPECT(total > 0);
}

static void test_errors() {
  const int d = 16;
  std::vector<float> xb = random_rows(8, d, 8), xq = random_rows(2, d, 9);
  const auto queries = to_pb(xq, {0, 0}, d);
  {  // a repeated id inside one batch: EVECTOR_ID_DUPLICATED, the batch adds nothing, the scan goes on
    for (bool with_host_filter : {false, true}) {
      Filters fs;
      if (with_host_filter) fs.push_back(std::make_shared<FnFilter>([](int64_t id) { return id != 3; }));
      BruteForceRangeScannerB200 sc(pb::common::METRIC_TYPE_L2, d, queries, 1e9f, fs);
      auto st = sc.Push(to_pb(xb, {1, 2, 3, 3}, d));
      EXPECT(!st.ok() && st.error_code() == pb::error::EVECTOR_ID_DUPLICATED);
      EXPECT(sc.Push(to_pb(std::vector<float>(xb.begin() + 4 * d, xb.end()), {5, 6, 7, 8}, d)).ok());
      Results got;
      EXPECT(sc.Finish(got).ok());
      EXPECT(got.size() == 2 && got[0].vector_with_distances_size() == 4 && got[0].vector_with_distances(0).vector_with_id().id() == 5);
    }
  }
  {  // a batch row of the wrong dimension
    BruteForceRangeScannerB200 sc(pb::common::METRIC_TYPE_L2, d, queries, 1.0f, {});
    auto bad = to_pb(std::vector<float>(xb.begin(), xb.begin() + 8), {1}, 8);
    auto st = sc.Push(bad);
    EXPECT(!st.ok() && st.error_code() == pb::error::EVECTOR_INVALID);
  }
  {
    BruteForceRangeScannerB200 sc(pb::common::METRIC_TYPE_L2, 0, queries, 1.0f, {});
    Results got;
    auto st = sc.Finish(got);
    EXPECT(!st.ok() && st.error_code() == pb::error::EVECTOR_INVALID);
  }
  {
    BruteForceRangeScannerB200 sc(pb::common::METRIC_TYPE_L2, d, {}, 1.0f, {});
    Results got;
    auto st = sc.Finish(got);
    EXPECT(!st.ok() && st.error_code() == pb::error::EILLEGAL_PARAMTETERS);
  }
  {  // nothing pushed: one empty result per query
    BruteForceRangeScannerB200 sc(pb::common::METRIC_TYPE_L2, d, queries, 1.0f, {});
    Results got;
    EXPECT(sc.Finish(got).ok());
    EXPECT(got.size() == 2 && got[0].vector_with_distances_size() == 0 && got[1].vector_with_distances_size() == 0);
  }
}

int main() {
  {
    std::vector<float> q = random_rows(1, 8, 0);
    b200vs_scan_range* h = nullptr;
    if (b200vs_scan_range_begin(0, B200VS_L2, 8, 1, q.data(), 1.0f, 1, nullptr, &h) != B200VS_OK) {
      printf("cannot begin a scan: %s\n", b200vs_last_error());  // no CUDA device: the product has no CPU fallback
      return 2;
    }
    b200vs_scan_range_abort(h);
  }
  test_filters_l2();
  test_cap_ip();
  test_cosine_matches_flat_range_search();
  test_errors();
  if (g_fail) { printf("%d FAILURES\n", g_fail); return 1; }
  printf("PLUGIN SCAN RANGE TESTS OK\n");
  return 0;
}
