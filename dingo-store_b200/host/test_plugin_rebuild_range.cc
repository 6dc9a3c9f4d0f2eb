// test_plugin_rebuild_range.cc — the plugin's split and merge rebuilds: RebuildFrom(olds, min, max) gives an index whose Search
// results, with no range filter, equal a fresh Train + Add of the rows with min <= id < max of olds in ascending id order, so
// a split parent never returns its child's rows; its refusals come back as the reference's error codes.  Needs a GPU; run by
// tests/test_gpu_plugin_rebuild_range.py.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <numeric>
#include <random>
#include <vector>

#include "vector_index_b200.h"

using namespace dingodb;

static int g_fail = 0;
#define EXPECT(cond)                                                                \
  do {                                                                              \
    if (!(cond)) { ++g_fail; printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); } \
  } while (0)

static const int kDim = 32, kNlist = 8, kTopk = 50;
using Ix = std::shared_ptr<VectorIndexB200>;

static std::vector<float> fixture(int n, unsigned seed) {
  std::mt19937 rng(seed);
  std::normal_distribution<float> nd;
  std::vector<float> x((size_t)n * kDim);
  for (auto& v : x) v = nd(rng);
  return x;
}
static std::vector<pb::common::VectorWithId> to_pb(const std::vector<float>& x, const std::vector<int64_t>& ids) {
  std::vector<pb::common::VectorWithId> out(ids.size());
  for (size_t i = 0; i < ids.size(); ++i) {
    out[i].set_id(ids[i]);
    out[i].mutable_vector()->set_dimension(kDim);
    out[i].mutable_vector()->set_value_type(pb::common::ValueType::FLOAT);
    for (int j = 0; j < kDim; ++j) out[i].mutable_vector()->add_float_values(x[i * kDim + j]);
  }
  return out;
}
static Ix make(pb::common::VectorIndexType type) {
  pb::common::VectorIndexParameter p;
  p.set_vector_index_type(type);
  if (type == pb::common::VECTOR_INDEX_TYPE_IVF_FLAT) {
    auto* q = p.mutable_ivf_flat_parameter();
    q->dimension_ = kDim; q->metric_type_ = pb::common::METRIC_TYPE_L2; q->ncentroids_ = kNlist;
  } else if (type == pb::common::VECTOR_INDEX_TYPE_FLAT) {
    auto* q = p.mutable_flat_parameter();
    q->dimension_ = kDim; q->metric_type_ = pb::common::METRIC_TYPE_L2;
  } else {
    auto* q = p.mutable_hnsw_parameter();
    q->dimension_ = kDim; q->metric_type_ = pb::common::METRIC_TYPE_L2; q->nlinks_ = 8; q->efconstruction_ = 40; q->max_elements_ = 10000;
  }
  return std::make_shared<VectorIndexB200>(1, p, pb::common::RegionEpoch(), pb::common::Range(), nullptr);
}
// top-kTopk of every query over every list, with no filter
static void search(const Ix& ix, const std::vector<pb::common::VectorWithId>& qs, std::vector<int64_t>& ids, std::vector<float>& dist) {
  pb::common::VectorSearchParameter sp;
  sp.mutable_ivf_flat()->set_nprobe(kNlist);
  std::vector<pb::index::VectorWithDistanceResult> results;
  EXPECT(ix->Search(qs, kTopk, {}, false, sp, results).ok());
  ids.assign(qs.size() * kTopk, -1);
  dist.assign(qs.size() * kTopk, 0.f);
  for (size_t q = 0; q < results.size() && q < qs.size(); ++q)
    for (int i = 0; i < results[q].vector_with_distances_size() && i < kTopk; ++i) {
      ids[q * kTopk + i] = results[q].vector_with_distances(i).vector_with_id().id();
      dist[q * kTopk + i] = results[q].vector_with_distances(i).distance();
    }
}

// A region's rows: ids given out of order, row i of x under ids[i]
struct Rows {
  std::vector<int64_t> ids;
  std::vector<float> x;
};
static Rows region(int64_t first, int n, unsigned seed) {
  Rows r;
  r.ids.resize(n);
  std::iota(r.ids.begin(), r.ids.end(), first);
  std::shuffle(r.ids.begin(), r.ids.end(), std::mt19937(seed));
  r.x = fixture(n, seed + 1);
  return r;
}
// a fresh index trained and filled with the rows of parts with lo <= id < hi in ascending id order
static Ix fresh(pb::common::VectorIndexType type, const std::vector<const Rows*>& parts, int64_t lo, int64_t hi) {
  std::vector<std::pair<int64_t, const float*>> sel;
  for (const Rows* p : parts)
    for (size_t i = 0; i < p->ids.size(); ++i)
      if (p->ids[i] >= lo && p->ids[i] < hi) sel.emplace_back(p->ids[i], p->x.data() + i * kDim);
  std::sort(sel.begin(), sel.end());
  std::vector<float> xs(sel.size() * kDim);
  std::vector<int64_t> ids(sel.size());
  for (size_t i = 0; i < sel.size(); ++i) {
    ids[i] = sel[i].first;
    std::copy(sel[i].second, sel[i].second + kDim, xs.begin() + i * kDim);
  }
  Ix f = make(type);
  if (type == pb::common::VECTOR_INDEX_TYPE_IVF_FLAT) {
    std::vector<float> t = xs;
    EXPECT(f->Train(t).ok());
  }
  EXPECT(f->Add(to_pb(xs, ids)).ok());
  return f;
}
static bool same_reads(const Ix& a, const Ix& b, const std::vector<pb::common::VectorWithId>& qs) {
  std::vector<int64_t> ia, ib;
  std::vector<float> da, db;
  search(a, qs, ia, da);
  search(b, qs, ib, db);
  return ia == ib && da == db;
}

int main() {
  const auto qs = to_pb(fixture(16, 3), std::vector<int64_t>(16, 0));
  for (auto type : {pb::common::VECTOR_INDEX_TYPE_IVF_FLAT, pb::common::VECTOR_INDEX_TYPE_FLAT}) {
    // ---- split at s: the child takes [s, end) from the parent's index as its share index, the parent keeps [0, s) ----
    const int64_t s = 1300;
    const Rows par = region(0, 3000, 7);
    Ix old = make(type);
    if (type == pb::common::VECTOR_INDEX_TYPE_IVF_FLAT) {
      std::vector<float> t(par.x.begin(), par.x.begin() + 500 * kDim);
      EXPECT(old->Train(t).ok());
    }
    EXPECT(old->Add(to_pb(par.x, par.ids)).ok());
    Ix parent = make(type), child = make(type);
    EXPECT(parent->RebuildFrom({old.get()}, 0, s).ok());
    EXPECT(child->RebuildFrom({old.get()}, s, INT64_MAX).ok());
    int64_t cp = 0, cc = 0;
    EXPECT(parent->GetCount(cp).ok() && cp == s && child->GetCount(cc).ok() && cc == 3000 - s);
    std::vector<int64_t> ids;
    std::vector<float> dist;
    search(parent, qs, ids, dist);  // no range filter: the index range equals the region range
    EXPECT(std::count(ids.begin(), ids.end(), -1) == 0);
    EXPECT(std::all_of(ids.begin(), ids.end(), [&](int64_t id) { return id >= 0 && id < s; }));
    search(child, qs, ids, dist);
    EXPECT(std::all_of(ids.begin(), ids.end(), [&](int64_t id) { return id >= s; }));
    EXPECT(same_reads(parent, fresh(type, {&par}, 0, s), qs));
    EXPECT(same_reads(child, fresh(type, {&par}, s, INT64_MAX), qs));

    // ---- merge: the target's own index and the sibling, each also holding rows outside the merged range ----
    const Rows a = region(0, 2000, 11), b = region(2000, 2000, 13);
    Ix own = make(type), sib = make(type);
    for (auto& [ix, r] : {std::pair<Ix, const Rows*>{own, &a}, {sib, &b}}) {
      if (type == pb::common::VECTOR_INDEX_TYPE_IVF_FLAT) {
        std::vector<float> t(r->x.begin(), r->x.begin() + 300 * kDim);
        EXPECT(ix->Train(t).ok());
      }
      EXPECT(ix->Add(to_pb(r->x, r->ids)).ok());
    }
    Ix merged = make(type);
    EXPECT(merged->RebuildFrom({own.get(), sib.get()}, 500, 3500).ok());
    int64_t cm = 0;
    EXPECT(merged->GetCount(cm).ok() && cm == 3000);
    search(merged, qs, ids, dist);
    EXPECT(std::all_of(ids.begin(), ids.end(), [&](int64_t id) { return id >= 500 && id < 3500; }));
    EXPECT(same_reads(merged, fresh(type, {&a, &b}, 500, 3500), qs));

    // ---- refusals, as pb codes; the sources keep serving the same results ----
    std::vector<int64_t> i0, i1;
    std::vector<float> d0, d1;
    search(old, qs, i0, d0);
    EXPECT(parent->RebuildFrom({old.get()}, 0, s).error_code() == pb::error::EILLEGAL_PARAMTETERS);       // dst not empty
    EXPECT(make(type)->RebuildFrom({}, 0, s).error_code() == pb::error::EILLEGAL_PARAMTETERS);              // no source
    EXPECT(make(type)->RebuildFrom({old.get(), old.get()}, 0, s).error_code() == pb::error::EILLEGAL_PARAMTETERS);  // twice
    EXPECT(make(type)->RebuildFrom({old.get(), nullptr}, 0, s).error_code() == pb::error::EILLEGAL_PARAMTETERS);  // null
    EXPECT(make(type)->RebuildFrom({old.get()}, s, 0).error_code() == pb::error::EILLEGAL_PARAMTETERS);     // min > max
    EXPECT(make(pb::common::VECTOR_INDEX_TYPE_HNSW)->RebuildFrom({old.get()}, 0, s).error_code() == pb::error::EILLEGAL_PARAMTETERS);
    EXPECT(old->RebuildFrom({old.get()}, 0, s).error_code() == pb::error::EILLEGAL_PARAMTETERS);           // dst a source
    EXPECT(make(type)->RebuildFrom({old.get(), own.get()}, 0, 3000).error_code() == pb::error::EVECTOR_ID_DUPLICATED);
    search(old, qs, i1, d1);
    EXPECT(i0 == i1 && d0 == d1);
    // an empty range: OK, nothing copied
    Ix empty = make(type);
    int64_t ce = -1;
    EXPECT(empty->RebuildFrom({old.get()}, 5000, 6000).ok() && empty->GetCount(ce).ok() && ce == 0);
    EXPECT(type != pb::common::VECTOR_INDEX_TYPE_IVF_FLAT || !empty->IsTrained());
  }

  if (g_fail) { printf("%d FAILURES\n", g_fail); return 1; }
  printf("PLUGIN REBUILD RANGE TESTS OK\n");
  return 0;
}
