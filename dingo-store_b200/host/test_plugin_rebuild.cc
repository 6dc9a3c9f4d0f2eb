// test_plugin_rebuild.cc — the plugin's rebuild surface: NeedToRebuild() follows b200vs_need_rebuild's rule, and RebuildFrom
// gives an index whose Search results equal a fresh Train + Add of the old index's live rows in ascending id order; its
// refusals come back as the reference's error codes.  Needs a GPU; run by tests/test_gpu_plugin_rebuild.py.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
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

static const int kDim = 32, kNlist = 8, kTopk = 10;

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
static std::shared_ptr<VectorIndexB200> make_ivf(int nlist = kNlist) {
  pb::common::VectorIndexParameter p;
  p.set_vector_index_type(pb::common::VECTOR_INDEX_TYPE_IVF_FLAT);
  auto* q = p.mutable_ivf_flat_parameter();
  q->dimension_ = kDim; q->metric_type_ = pb::common::METRIC_TYPE_L2; q->ncentroids_ = nlist;
  return std::make_shared<VectorIndexB200>(1, p, pb::common::RegionEpoch(), pb::common::Range(), nullptr);
}
static std::shared_ptr<VectorIndexB200> make_hnsw() {
  pb::common::VectorIndexParameter p;
  p.set_vector_index_type(pb::common::VECTOR_INDEX_TYPE_HNSW);
  auto* q = p.mutable_hnsw_parameter();
  q->dimension_ = kDim; q->metric_type_ = pb::common::METRIC_TYPE_L2; q->nlinks_ = 8; q->efconstruction_ = 40; q->max_elements_ = 1000;
  return std::make_shared<VectorIndexB200>(2, p, pb::common::RegionEpoch(), pb::common::Range(), nullptr);
}
static void search(std::shared_ptr<VectorIndexB200> ix, const std::vector<pb::common::VectorWithId>& qs, std::vector<int64_t>& ids,
                   std::vector<float>& dist) {
  pb::common::VectorSearchParameter sp;
  sp.mutable_ivf_flat()->set_nprobe(4);
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

int main() {
  // ---- IVF-Flat: the degenerate nlist = 1 region reaches 256 * nlist rows ----
  const int thr = 256 * kNlist;
  auto src = make_ivf();
  std::vector<float> tiny = fixture(5, 1);
  EXPECT(src->Train(tiny).ok());
  std::vector<int64_t> ids(thr);
  std::iota(ids.begin(), ids.end(), 100);
  std::shuffle(ids.begin(), ids.end(), std::mt19937(7));  // ids given out of order
  const std::vector<float> x = fixture(thr, 2);
  std::vector<int64_t> first(ids.begin(), ids.end() - 1);
  EXPECT(src->Add(to_pb(x, first)).ok());
  EXPECT(!src->NeedToRebuild());
  std::vector<float> last(x.end() - kDim, x.end());
  EXPECT(src->Add(to_pb(last, {ids.back()})).ok());
  EXPECT(src->NeedToRebuild());
  EXPECT(src->Delete({ids[0]}).ok());  // one row below the threshold again
  EXPECT(!src->NeedToRebuild());
  EXPECT(src->Add(to_pb(std::vector<float>(x.begin(), x.begin() + kDim), {ids[0]})).ok());
  EXPECT(src->NeedToRebuild());

  // ---- RebuildFrom equals a fresh Train + Add of the live rows in ascending id order ----
  auto dst = make_ivf();
  EXPECT(dst->RebuildFrom(*src).ok());
  EXPECT(dst->IsTrained() && !dst->NeedToRebuild());  // trained on every row: train_rows == count
  int64_t c_src = 0, c_dst = 0;
  EXPECT(src->GetCount(c_src).ok() && dst->GetCount(c_dst).ok() && c_src == c_dst && c_dst == thr);
  std::vector<size_t> order(thr);
  std::iota(order.begin(), order.end(), 0);
  std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return ids[a] < ids[b]; });
  std::vector<float> xs((size_t)thr * kDim);
  std::vector<int64_t> sids(thr);
  for (int i = 0; i < thr; ++i) {
    sids[i] = ids[order[i]];
    std::copy(x.begin() + order[i] * kDim, x.begin() + (order[i] + 1) * kDim, xs.begin() + (size_t)i * kDim);
  }
  auto fresh = make_ivf();
  std::vector<float> xs_train = xs;
  EXPECT(fresh->Train(xs_train).ok());
  EXPECT(fresh->Add(to_pb(xs, sids)).ok());
  const auto qs = to_pb(fixture(16, 3), std::vector<int64_t>(16, 0));
  std::vector<int64_t> i_dst, i_fresh, i_src, i_src_after;
  std::vector<float> d_dst, d_fresh, d_src, d_src_after;
  search(dst, qs, i_dst, d_dst);
  search(fresh, qs, i_fresh, d_fresh);
  EXPECT(i_dst == i_fresh && d_dst == d_fresh);
  EXPECT(std::count(i_dst.begin(), i_dst.end(), -1) == 0);

  // ---- refusals keep both indexes as they were, as the reference's error codes ----
  search(src, qs, i_src, d_src);
  EXPECT(dst->RebuildFrom(*src).error_code() == pb::error::EILLEGAL_PARAMTETERS);  // dst not empty
  EXPECT(make_ivf(kNlist * 2)->RebuildFrom(*src).error_code() == pb::error::EILLEGAL_PARAMTETERS);  // another nlist
  EXPECT(make_hnsw()->RebuildFrom(*src).error_code() == pb::error::EILLEGAL_PARAMTETERS);  // another type
  search(src, qs, i_src_after, d_src_after);
  EXPECT(i_src == i_src_after && d_src == d_src_after);
  search(dst, qs, i_src_after, d_src_after);
  EXPECT(i_src_after == i_dst && d_src_after == d_dst);

  // ---- HNSW: tombstones more than half of every node ----
  auto h = make_hnsw();
  std::vector<int64_t> hid(300);
  std::iota(hid.begin(), hid.end(), 1);
  EXPECT(h->Add(to_pb(fixture(300, 4), hid)).ok());
  EXPECT(!h->NeedToRebuild());
  EXPECT(h->Delete(std::vector<int64_t>(hid.begin(), hid.begin() + 150)).ok());
  EXPECT(!h->NeedToRebuild());  // 150 of 300: not more than half
  EXPECT(h->Delete({151}).ok());
  EXPECT(h->NeedToRebuild());
  auto h2 = make_hnsw();
  EXPECT(h2->RebuildFrom(*h).ok() && !h2->NeedToRebuild());
  int64_t hc = 0, hdel = -1;
  EXPECT(h2->GetCount(hc).ok() && hc == 149 && h2->GetDeletedCount(hdel).ok() && hdel == 0);

  if (g_fail) { printf("%d FAILURES\n", g_fail); return 1; }
  printf("PLUGIN REBUILD TESTS OK\n");
  return 0;
}
