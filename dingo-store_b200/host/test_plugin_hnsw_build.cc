// test_plugin_hnsw_build.cc — the plugin's HNSW device build (VectorIndexB200::hnsw_device_build_min_rows): an Add of at
// least that many rows builds the graph with b200vs_hnsw_add_batched, a smaller one keeps the host builder.  Needs a GPU; run
// by tests/test_gpu_plugin_hnsw_build.py.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <random>
#include <string>

#include <unistd.h>

#include "vector_index_b200.h"

using namespace dingodb;

static int g_fail = 0;
#define EXPECT(cond)                                                                \
  do {                                                                              \
    if (!(cond)) { ++g_fail; printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); } \
  } while (0)

static const int kDim = 32, kM = 16, kEfc = 200, kEf = 64, kTopk = 10;

static std::vector<float> fixture(int n, int d, unsigned seed) {
  std::mt19937 rng(seed);
  std::uniform_real_distribution<> distrib;
  std::vector<float> x((size_t)n * d);
  for (auto& v : x) v = (float)distrib(rng);
  return x;
}
static std::vector<pb::common::VectorWithId> to_pb(const std::vector<float>& x, int n, int d, int64_t first_id) {
  std::vector<pb::common::VectorWithId> out(n);
  for (int i = 0; i < n; ++i) {
    out[i].set_id(first_id + i);
    out[i].mutable_vector()->set_dimension(d);
    out[i].mutable_vector()->set_value_type(pb::common::ValueType::FLOAT);
    for (int j = 0; j < d; ++j) out[i].mutable_vector()->add_float_values(x[(size_t)i * d + j]);
  }
  return out;
}
static VectorIndexPtr make_plugin() {
  pb::common::VectorIndexParameter p;
  p.set_vector_index_type(pb::common::VECTOR_INDEX_TYPE_HNSW);
  auto* q = p.mutable_hnsw_parameter();
  q->dimension_ = kDim; q->metric_type_ = pb::common::METRIC_TYPE_L2; q->nlinks_ = kM; q->efconstruction_ = kEfc; q->max_elements_ = 10000;
  auto ix = std::make_shared<VectorIndexB200>(1, p, pb::common::RegionEpoch(), pb::common::Range(), nullptr);
  int64_t c = 0;
  if (!ix->GetCount(c).ok()) {
    printf("cannot create the index: %s\n", b200vs_last_error());
    exit(2);
  }
  return ix;
}
// ids[q * k + i], dist[q * k + i] of a plugin search
static void plugin_search(VectorIndexPtr ix, const std::vector<pb::common::VectorWithId>& qs, std::vector<int64_t>& ids, std::vector<float>& dist) {
  pb::common::VectorSearchParameter sp;
  sp.mutable_hnsw()->set_efsearch(kEf);
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

// the bytes of an index file (Save / b200vs_save: the graph, the rows and the labels)
static std::string slurp(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  return std::string(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}
static std::string tmp_path(const char* name) {
  const char* dir = getenv("TMPDIR");
  return std::string(dir && *dir ? dir : "/tmp") + "/b200vs_hnsw_build_" + std::to_string((long)getpid()) + "_" + name;
}
static b200vs_index* abi_index() {
  b200vs_params bp;
  memset(&bp, 0, sizeof(bp));
  bp.hnsw_m = kM; bp.hnsw_efc = kEfc; bp.max_elements = 10000;
  b200vs_index* abi = nullptr;
  EXPECT(b200vs_create(B200VS_HNSW, B200VS_L2, kDim, &bp, &abi) == B200VS_OK);
  return abi;
}
// the file of an ABI index holding rows x with ids 1.. (device: b200vs_hnsw_add_batched, default batch; else the host builder)
static std::string abi_file(const std::vector<float>& x, int n, int64_t first_id, bool device, const char* name) {
  b200vs_index* abi = abi_index();
  std::vector<int64_t> ids(n);
  for (int i = 0; i < n; ++i) ids[i] = first_id + i;
  EXPECT((device ? b200vs_hnsw_add_batched(abi, n, x.data(), ids.data(), 0) : b200vs_add_with_ids(abi, n, x.data(), ids.data(), 0)) == B200VS_OK);
  const std::string path = tmp_path(name);
  EXPECT(b200vs_save(abi, path.c_str()) == B200VS_OK);
  b200vs_destroy(abi);
  std::string bytes = slurp(path);
  remove(path.c_str());
  return bytes;
}
static std::string plugin_file(VectorIndexPtr ix, const char* name) {
  const std::string path = tmp_path(name);
  EXPECT(ix->Save(path).ok());
  std::string bytes = slurp(path);
  remove(path.c_str());
  return bytes;
}

static void test_large_add_builds_on_device() {
  const int n = 5000, nq = 20;
  auto x = fixture(n, kDim, 1);
  auto xq = fixture(nq, kDim, 2);
  VectorIndexB200::hnsw_device_build_min_rows = 1000;
  auto ix = make_plugin();
  EXPECT(ix->Add(to_pb(x, n, kDim, 1)).ok());
  std::vector<int64_t> pi;
  std::vector<float> pd;
  plugin_search(ix, to_pb(xq, nq, kDim, 0), pi, pd);
  VectorIndexB200::hnsw_device_build_min_rows = 0;
  // the plugin's graph is the batched one, and on these rows the batched and host graphs differ
  const std::string got = plugin_file(ix, "plugin"), dev = abi_file(x, n, 1, true, "dev"), host = abi_file(x, n, 1, false, "host");
  EXPECT(!got.empty() && got == dev);
  EXPECT(dev != host);

  b200vs_index* abi = abi_index();
  std::vector<int64_t> ids(n);
  for (int i = 0; i < n; ++i) ids[i] = i + 1;
  EXPECT(b200vs_hnsw_add_batched(abi, n, x.data(), ids.data(), 0) == B200VS_OK);
  b200vs_search_params sp;
  memset(&sp, 0, sizeof(sp));
  sp.efsearch = kEf;
  std::vector<int64_t> ai((size_t)nq * kTopk);
  std::vector<float> ad((size_t)nq * kTopk);
  EXPECT(b200vs_search(abi, nq, xq.data(), kTopk, &sp, ad.data(), ai.data()) == B200VS_OK);
  EXPECT(ai == pi);
  EXPECT(memcmp(ad.data(), pd.data(), ad.size() * sizeof(float)) == 0);
  int64_t count = 0;
  EXPECT(ix->GetCount(count).ok() && count == n);
  b200vs_destroy(abi);
}

static void test_small_add_keeps_host_builder() {
  const int n = 10;
  auto x = fixture(n, kDim, 3);
  auto vs = to_pb(x, n, kDim, 100);
  auto qs = to_pb(fixture(4, kDim, 4), 4, kDim, 0);
  VectorIndexB200::hnsw_device_build_min_rows = 1000;
  auto on = make_plugin();
  EXPECT(on->Add(vs).ok());
  std::vector<int64_t> i1, i2;
  std::vector<float> d1, d2;
  plugin_search(on, qs, i1, d1);
  VectorIndexB200::hnsw_device_build_min_rows = 0;
  auto off = make_plugin();
  EXPECT(off->Add(vs).ok());
  plugin_search(off, qs, i2, d2);
  EXPECT(i1 == i2);
  EXPECT(memcmp(d1.data(), d2.data(), d1.size() * sizeof(float)) == 0);
  EXPECT(i1[0] >= 100);
  // both are the host builder's graph
  const std::string a = plugin_file(on, "on"), b = plugin_file(off, "off");
  EXPECT(!a.empty() && a == b && a == abi_file(x, n, 100, false, "host10"));
}

int main() {
  test_large_add_builds_on_device();
  test_small_add_keeps_host_builder();
  if (g_fail) {
    printf("%d failures\n", g_fail);
    return 1;
  }
  printf("PLUGIN HNSW BUILD TESTS OK\n");
  return 0;
}
