// test_plugin_deep.cc — VectorIndexB200::Search above the service's top_n limit: topk > 4096 (the reader's scalar post-filter
// over-fetch, vector_reader.cc:119-215) goes to b200vs_search_deep / b200vs_search_binary_deep on Flat, IVF-Flat, IVF-PQ and
// Binary Flat, and topk <= 4096 to b200vs_search / b200vs_search_binary as before.  Every plugin search is compared, hit by
// hit, with the direct ABI call on an index built from the same rows; HNSW keeps b200vs_search's refusal.
// Needs a GPU; run by tests/test_gpu_deep_topk.py.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>

#include "vector_index_b200.h"

using namespace dingodb;
using Results = std::vector<pb::index::VectorWithDistanceResult>;

static int g_fail = 0;
#define EXPECT(cond)                                                                \
  do {                                                                              \
    if (!(cond)) { ++g_fail; printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); } \
  } while (0)

struct Rows {
  int n, dim;        // dim: floats, or bits of a binary row
  bool binary;
  std::vector<float> x;
  std::vector<uint8_t> xb;
  std::vector<int64_t> ids;
};

static Rows make_rows(int n, int dim, bool binary, unsigned seed) {
  Rows r{n, dim, binary, {}, {}, {}};
  std::mt19937 rng(seed);
  std::normal_distribution<float> nd;
  if (binary) { r.xb.resize((size_t)n * dim / 8); for (auto& b : r.xb) b = (uint8_t)(rng() & 0xFF); }
  else { r.x.resize((size_t)n * dim); for (auto& v : r.x) v = nd(rng); }
  r.ids.resize(n);
  for (int i = 0; i < n; ++i) r.ids[i] = 3 * (int64_t)i + 1;
  return r;
}

static std::vector<pb::common::VectorWithId> to_pb(const Rows& r, int first, int count) {
  std::vector<pb::common::VectorWithId> out(count);
  const int nb = r.dim / 8;
  for (int i = 0; i < count; ++i) {
    const int row = first + i;
    out[i].set_id(r.ids[row]);
    auto* v = out[i].mutable_vector();
    v->set_dimension(r.dim);
    if (r.binary) {
      v->set_value_type(pb::common::ValueType::UINT8);
      for (int j = 0; j < nb; ++j) v->add_binary_values(std::string(1, (char)r.xb[(size_t)row * nb + j]));
    } else {
      v->set_value_type(pb::common::ValueType::FLOAT);
      for (int j = 0; j < r.dim; ++j) v->add_float_values(r.x[(size_t)row * r.dim + j]);
    }
  }
  return out;
}

struct Case {
  const char* name;
  pb::common::VectorIndexType t;
  b200vs_type bt;
  pb::common::MetricType m;
  b200vs_metric bm;
  int dim, nlist, pq_m, pq_nbits;
  bool binary;
};

static void run_case(const Case& c, int n) {
  printf("-- %s\n", c.name);
  const Rows r = make_rows(n, c.dim, c.binary, 7);
  pb::common::VectorIndexParameter p;
  p.set_vector_index_type(c.t);
  if (c.t == pb::common::VECTOR_INDEX_TYPE_FLAT) { auto* q = p.mutable_flat_parameter(); q->dimension_ = c.dim; q->metric_type_ = c.m; }
  if (c.t == pb::common::VECTOR_INDEX_TYPE_IVF_FLAT) { auto* q = p.mutable_ivf_flat_parameter(); q->dimension_ = c.dim; q->metric_type_ = c.m; q->ncentroids_ = c.nlist; }
  if (c.t == pb::common::VECTOR_INDEX_TYPE_IVF_PQ) {
    auto* q = p.mutable_ivf_pq_parameter();
    q->dimension_ = c.dim; q->metric_type_ = c.m; q->ncentroids_ = c.nlist; q->nsubvector_ = c.pq_m; q->nbits_per_idx_ = c.pq_nbits;
  }
  if (c.t == pb::common::VECTOR_INDEX_TYPE_BINARY_FLAT) { auto* q = p.mutable_binary_flat_parameter(); q->dimension_ = c.dim; q->metric_type_ = c.m; }
  auto ix = std::make_shared<VectorIndexB200>(1, p, pb::common::RegionEpoch(), pb::common::Range(), nullptr);
  int64_t cnt = 0;
  if (!ix->GetCount(cnt).ok()) {  // no CUDA device / library failure: the product has no CPU fallback, so neither has this test
    printf("cannot create the index: %s\n", b200vs_last_error());
    exit(2);
  }
  EXPECT(ix->Add(to_pb(r, 0, n)).ok());  // an untrained IVF index trains with the batch (ivf_flat.cc:133-150)

  // the same rows through the ABI: one train with the same batch, one add
  b200vs_params bp{};
  bp.nlist = c.nlist; bp.pq_m = c.pq_m; bp.pq_nbits = c.pq_nbits;
  b200vs_index* h = nullptr;
  EXPECT(b200vs_create(c.bt, c.bm, c.dim, &bp, &h) == B200VS_OK);
  if (c.nlist > 0) EXPECT(b200vs_train(h, n, r.x.data()) == B200VS_OK);
  if (c.binary) EXPECT(b200vs_add_with_ids_binary(h, n, r.xb.data(), r.ids.data(), 0) == B200VS_OK);
  else EXPECT(b200vs_add_with_ids(h, n, r.x.data(), r.ids.data(), 0) == B200VS_OK);

  const int nq = 2;
  const Rows qr = make_rows(nq, c.dim, c.binary, 11);
  const auto qs = to_pb(qr, 0, nq);
  pb::common::VectorSearchParameter sp;
  sp.mutable_ivf_flat()->set_nprobe(3);
  sp.mutable_ivf_pq()->set_nprobe(3);
  b200vs_search_params dsp{};
  dsp.nprobe = 3;
  for (uint32_t topk : {100u, 4096u, 4097u, 5000u, 40960u}) {
    Results res;
    EXPECT(ix->Search(qs, topk, {}, false, sp, res).ok());
    EXPECT(res.size() == (size_t)nq);
    std::vector<float> D((size_t)nq * topk);
    std::vector<int64_t> I((size_t)nq * topk);
    const bool deep = topk > 4096;
    int rc;
    if (c.binary) rc = (deep ? b200vs_search_binary_deep : b200vs_search_binary)(h, nq, qr.xb.data(), (int32_t)topk, &dsp, D.data(), I.data());
    else rc = (deep ? b200vs_search_deep : b200vs_search)(h, nq, qr.x.data(), (int32_t)topk, &dsp, D.data(), I.data());
    EXPECT(rc == B200VS_OK);
    int bad = 0;
    for (int q = 0; q < nq && q < (int)res.size(); ++q) {
      int hits = 0;
      for (uint32_t i = 0; i < topk; ++i) hits += I[(size_t)q * topk + i] >= 0;
      if (res[q].vector_with_distances_size() != hits) { ++bad; continue; }
      for (int i = 0; i < hits; ++i) {
        const auto& vd = res[q].vector_with_distances(i);
        const float d = D[(size_t)q * topk + i], got = vd.distance();
        if (vd.vector_with_id().id() != I[(size_t)q * topk + i] || std::memcmp(&d, &got, 4) != 0) ++bad;
      }
    }
    printf("   topk %u: %d mismatches\n", topk, bad);
    EXPECT(bad == 0);
  }
  b200vs_destroy(h);
}

static void test_hnsw_refusal() {
  printf("-- HNSW\n");
  const int n = 300, d = 16;
  const Rows r = make_rows(n, d, false, 5);
  pb::common::VectorIndexParameter p;
  p.set_vector_index_type(pb::common::VECTOR_INDEX_TYPE_HNSW);
  auto* q = p.mutable_hnsw_parameter();
  q->dimension_ = d; q->metric_type_ = pb::common::METRIC_TYPE_L2; q->nlinks_ = 16; q->efconstruction_ = 64; q->max_elements_ = 1000;
  auto ix = std::make_shared<VectorIndexB200>(1, p, pb::common::RegionEpoch(), pb::common::Range(), nullptr);
  EXPECT(ix->Add(to_pb(r, 0, n)).ok());
  b200vs_params bp{};
  bp.hnsw_m = 16; bp.hnsw_efc = 64; bp.max_elements = 1000;
  b200vs_index* h = nullptr;
  EXPECT(b200vs_create(B200VS_HNSW, B200VS_L2, d, &bp, &h) == B200VS_OK);
  EXPECT(b200vs_add_with_ids(h, n, r.x.data(), r.ids.data(), 0) == B200VS_OK);
  const auto qs = to_pb(r, 0, 1);
  pb::common::VectorSearchParameter sp;
  for (uint32_t topk : {5000u, 40960u}) {
    Results res;
    const auto st = ix->Search(qs, topk, {}, false, sp, res);
    std::vector<float> D(topk);
    std::vector<int64_t> I(topk);
    const int rc = b200vs_search(h, 1, r.x.data(), (int32_t)topk, nullptr, D.data(), I.data());
    // HNSW stays on b200vs_search: the plugin answers or refuses as the ABI does, and the walk's shared memory refuses 40960
    EXPECT((rc == B200VS_OK) == st.ok());
    EXPECT(rc != B200VS_EILLEGAL_PARAMETERS || st.error_code() == pb::error::EILLEGAL_PARAMTETERS);
    EXPECT(topk < 40960 || rc != B200VS_OK);
    printf("   topk %u: rc %d, plugin error %d\n", topk, rc, (int)st.error_code());
  }
  Results res;
  EXPECT(ix->Search(qs, 10, {}, false, sp, res).ok() && res.size() == 1 && res[0].vector_with_distances_size() == 10);
  b200vs_destroy(h);
}

int main() {
  const Case cases[] = {
      {"FLAT L2", pb::common::VECTOR_INDEX_TYPE_FLAT, B200VS_FLAT, pb::common::METRIC_TYPE_L2, B200VS_L2, 32, 0, 0, 0, false},
      {"FLAT IP", pb::common::VECTOR_INDEX_TYPE_FLAT, B200VS_FLAT, pb::common::METRIC_TYPE_INNER_PRODUCT, B200VS_IP, 32, 0, 0, 0, false},
      {"IVF_FLAT L2", pb::common::VECTOR_INDEX_TYPE_IVF_FLAT, B200VS_IVF_FLAT, pb::common::METRIC_TYPE_L2, B200VS_L2, 32, 8, 0, 0, false},
      {"IVF_FLAT COSINE", pb::common::VECTOR_INDEX_TYPE_IVF_FLAT, B200VS_IVF_FLAT, pb::common::METRIC_TYPE_COSINE, B200VS_COSINE, 32, 8, 0, 0, false},
      // 4-bit codes: max(256 * nlist, 256 * 2^nbits) = 4096 training rows put the index in its IVF-PQ mode
      {"IVF_PQ L2", pb::common::VECTOR_INDEX_TYPE_IVF_PQ, B200VS_IVF_PQ, pb::common::METRIC_TYPE_L2, B200VS_L2, 32, 4, 8, 4, false},
      {"BINARY_FLAT", pb::common::VECTOR_INDEX_TYPE_BINARY_FLAT, B200VS_BINARY_FLAT, pb::common::METRIC_TYPE_HAMMING, B200VS_HAMMING, 256, 0, 0, 0, true},
  };
  for (const auto& c : cases) run_case(c, 60000);
  test_hnsw_refusal();
  if (g_fail) { printf("%d FAILURES\n", g_fail); return 1; }
  printf("PLUGIN DEEP TESTS OK\n");
  return 0;
}
