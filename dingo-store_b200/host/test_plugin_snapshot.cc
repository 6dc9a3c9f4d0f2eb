// test_plugin_snapshot.cc — snapshots of the drop-in subclass through the fork-based save of
// VectorIndexSnapshotManager::SaveVectorIndexSnapshot (vector_index_snapshot_manager.cc:500-700), replayed step by step for
// every plugin type: LockWrite, fork, Save in the child, UnlockWrite plus more writes in the parent, waitpid, then Load into
// a new index.  Also the switch's default (no save support, as before), the non-fork branch (Save in-process between
// LockWrite and UnlockWrite) and NeedToSave's per-type rule.  Needs a GPU; run by tests/test_gpu_plugin_snapshot.py.
#include <signal.h>
#include <sys/wait.h>
#include <unistd.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>
#include <random>
#include <string>
#include <thread>

#include "vector_index_b200.h"

using namespace dingodb;
using Results = std::vector<pb::index::VectorWithDistanceResult>;

static int g_fail = 0;
#define EXPECT(cond)                                                                \
  do {                                                                              \
    if (!(cond)) { ++g_fail; printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); } \
  } while (0)

struct Case {
  const char* name;
  pb::common::VectorIndexType type;
  pb::common::MetricType metric;
  int dim, nlist, M, nbits, n;
};

static bool binary(const Case& c) {
  return c.type == pb::common::VECTOR_INDEX_TYPE_BINARY_FLAT || c.type == pb::common::VECTOR_INDEX_TYPE_BINARY_IVF_FLAT;
}

static std::vector<pb::common::VectorWithId> rows(const Case& c, int n, int64_t first_id, unsigned seed) {
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> u(-1.f, 1.f);
  std::vector<pb::common::VectorWithId> out(n);
  for (int i = 0; i < n; ++i) {
    out[i].set_id(first_id + i);
    auto* v = out[i].mutable_vector();
    v->set_dimension(c.dim);
    if (binary(c)) {
      v->set_value_type(pb::common::ValueType::UINT8);
      for (int j = 0; j < c.dim / 8; ++j) v->add_binary_values(std::string(1, (char)(rng() & 0xFF)));
    } else {
      v->set_value_type(pb::common::ValueType::FLOAT);
      for (int j = 0; j < c.dim; ++j) v->add_float_values(u(rng));
    }
  }
  return out;
}

static VectorIndexPtr make(const Case& c) {
  pb::common::VectorIndexParameter p;
  p.set_vector_index_type(c.type);
  switch (c.type) {
    case pb::common::VECTOR_INDEX_TYPE_FLAT: { auto* q = p.mutable_flat_parameter(); q->dimension_ = c.dim; q->metric_type_ = c.metric; break; }
    case pb::common::VECTOR_INDEX_TYPE_IVF_FLAT: { auto* q = p.mutable_ivf_flat_parameter(); q->dimension_ = c.dim; q->metric_type_ = c.metric; q->ncentroids_ = c.nlist; break; }
    case pb::common::VECTOR_INDEX_TYPE_IVF_PQ: {
      auto* q = p.mutable_ivf_pq_parameter();
      q->dimension_ = c.dim; q->metric_type_ = c.metric; q->ncentroids_ = c.nlist; q->nsubvector_ = c.M; q->nbits_per_idx_ = c.nbits;
      break;
    }
    case pb::common::VECTOR_INDEX_TYPE_HNSW: {
      auto* q = p.mutable_hnsw_parameter();
      q->dimension_ = c.dim; q->metric_type_ = c.metric; q->nlinks_ = 16; q->efconstruction_ = 100; q->max_elements_ = 4 * c.n + 1000;
      break;
    }
    case pb::common::VECTOR_INDEX_TYPE_BINARY_FLAT: { auto* q = p.mutable_binary_flat_parameter(); q->dimension_ = c.dim; q->metric_type_ = c.metric; break; }
    case pb::common::VECTOR_INDEX_TYPE_BINARY_IVF_FLAT: {
      auto* q = p.mutable_binary_ivf_flat_parameter(); q->dimension_ = c.dim; q->metric_type_ = c.metric; q->ncentroids_ = c.nlist;
      break;
    }
    default: break;
  }
  auto ix = std::make_shared<VectorIndexB200>(1, p, pb::common::RegionEpoch(), pb::common::Range(), nullptr);
  int64_t cnt = 0;
  if (!ix->GetCount(cnt).ok()) {  // no CUDA device / library failure: the product has no CPU fallback, so neither has this test
    printf("cannot create the index: %s\n", b200vs_last_error());
    exit(2);
  }
  return ix;
}

static Results search(const VectorIndexPtr& ix, const std::vector<pb::common::VectorWithId>& q, int nprobe = 4) {
  pb::common::VectorSearchParameter sp;
  sp.mutable_ivf_flat()->set_nprobe(nprobe);
  sp.mutable_ivf_pq()->set_nprobe(nprobe);
  sp.mutable_binary_ivf_flat()->set_nprobe(nprobe);
  sp.mutable_hnsw()->set_efsearch(256);
  Results r;
  EXPECT(ix->Search(q, 10, {}, false, sp, r).ok());
  return r;
}

static bool same(const Results& a, const Results& b) {
  if (a.size() != b.size()) return false;
  for (size_t q = 0; q < a.size(); ++q) {
    if (a[q].vector_with_distances_size() != b[q].vector_with_distances_size()) return false;
    for (int i = 0; i < a[q].vector_with_distances_size(); ++i) {
      const auto& x = a[q].vector_with_distances(i);
      const auto& y = b[q].vector_with_distances(i);
      if (x.vector_with_id().id() != y.vector_with_id().id() || x.distance() != y.distance()) return false;
    }
  }
  return true;
}

static std::string bytes_of(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  return std::string(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}

// waitpid with a timeout; a child still running at the timeout is killed and reaped, so none is left behind
static int reap(pid_t pid, int timeout_s) {
  int st = 0;
  const auto until = std::chrono::steady_clock::now() + std::chrono::seconds(timeout_s);
  while (std::chrono::steady_clock::now() < until) {
    const pid_t r = waitpid(pid, &st, WNOHANG);
    if (r == pid) return WIFEXITED(st) ? WEXITSTATUS(st) : 128 + WTERMSIG(st);
    if (r < 0) return -1;
    std::this_thread::sleep_for(std::chrono::milliseconds(5));
  }
  kill(pid, SIGKILL);
  waitpid(pid, &st, 0);
  printf("child timed out\n");
  return -2;
}

static void test_case(const Case& c, const std::string& dir) {
  printf("case %s\n", c.name);
  const std::string ref = dir + "/" + c.name + ".ref", forked = dir + "/" + c.name + ".fork", inproc = dir + "/" + c.name + ".inproc";
  auto ix = make(c);
  const auto base = rows(c, c.n, 1, 7);
  EXPECT(!ix->NeedToSave(20000));  // empty (and untrained): nothing to save, switch on or off
  VectorIndexB200::support_fork_save = true;
  EXPECT(ix->SupportSave() && !ix->NeedToSave(20000));
  EXPECT(ix->Add(base).ok());
  std::vector<int64_t> dead;
  for (int64_t i = 3; i <= c.n; i += 7) dead.push_back(i);  // tombstones
  EXPECT(ix->Delete(dead).ok());
  EXPECT(ix->NeedToSave(20000) && !ix->NeedToSave(10000));
  const auto queries = rows(c, 5, 1 << 30, 11);
  const Results before = search(ix, queries);

  // the reference bytes: b200vs_save at this state
  VectorIndexB200::support_fork_save = false;
  EXPECT(!ix->SupportSave() && !ix->NeedToSave(20000));
  EXPECT(ix->Save(ref).ok());
  VectorIndexB200::support_fork_save = true;

  // SaveVectorIndexSnapshot's fork branch
  ix->LockWrite();
  const pid_t pid = fork();
  if (pid == 0) _exit(ix->Save(forked).ok() ? 0 : 1);
  ix->UnlockWrite();
  EXPECT(ix->Add(rows(c, 200, 1000000, 13)).ok());  // writes while the child runs do not reach its file
  EXPECT(ix->Delete({1, 2, 4}).ok());
  EXPECT(pid > 0 && reap(pid, 120) == 0);
  EXPECT(bytes_of(forked) == bytes_of(ref) && !bytes_of(ref).empty());

  auto back = make(c);
  EXPECT(back->Load(forked).ok());
  EXPECT(same(search(back, queries), before));
  int64_t n0 = 0, n1 = 0;
  auto from_ref = make(c);
  EXPECT(from_ref->Load(ref).ok());
  EXPECT(back->GetCount(n0).ok() && from_ref->GetCount(n1).ok() && n0 == n1);
  EXPECT(back->GetDeletedCount(n0).ok() && from_ref->GetDeletedCount(n1).ok() && n0 == n1);
  EXPECT(back->VectorIndexSubType() == from_ref->VectorIndexSubType());

  // the non-fork branch: Save in-process between LockWrite and UnlockWrite writes b200vs_save's bytes of the same state
  VectorIndexB200::support_fork_save = false;
  EXPECT(ix->Save(ref).ok());
  VectorIndexB200::support_fork_save = true;
  ix->LockWrite();
  EXPECT(ix->Save(inproc).ok());
  EXPECT(ix->Save("").error_code() == pb::error::EILLEGAL_PARAMTETERS);
  ix->UnlockWrite();
  EXPECT(bytes_of(inproc) == bytes_of(ref));
  // without LockWrite nothing is staged: Save takes b200vs_save
  EXPECT(ix->Save(inproc).ok() && bytes_of(inproc) == bytes_of(ref));
  VectorIndexB200::support_fork_save = false;
  for (const auto& p : {ref, forked, inproc}) unlink(p.c_str());
}

// with the switch off (the default) the plugin behaves as before: no save support, Save and Load through b200vs_save
static void test_default_off(const std::string& dir) {
  EXPECT(!VectorIndexB200::support_fork_save);
  const Case c{"default_flat", pb::common::VECTOR_INDEX_TYPE_FLAT, pb::common::METRIC_TYPE_L2, 16, 0, 0, 0, 500};
  auto ix = make(c);
  EXPECT(ix->Add(rows(c, c.n, 1, 3)).ok());
  EXPECT(!ix->SupportSave() && !ix->NeedToSave(20000));
  const std::string path = dir + "/default.idx";
  ix->LockWrite();
  EXPECT(ix->Save(path).ok());
  ix->UnlockWrite();
  EXPECT(ix->Save("").error_code() == pb::error::EINTERNAL);  // b200vs_save cannot open "", as before
  auto back = make(c);
  EXPECT(back->Load(path).ok());
  const auto q = rows(c, 3, 1 << 30, 5);
  EXPECT(same(search(back, q), search(ix, q)));
  unlink(path.c_str());
}

// NeedToSave's per-type rule on untrained and emptied indexes
static void test_need_to_save_edges() {
  VectorIndexB200::support_fork_save = true;
  const Case ivf{"ivf_untrained", pb::common::VECTOR_INDEX_TYPE_IVF_FLAT, pb::common::METRIC_TYPE_L2, 16, 4, 0, 0, 100};
  auto ix = make(ivf);
  std::vector<float> train(100 * 16, 0.5f);
  for (size_t i = 0; i < train.size(); ++i) train[i] = (float)(i % 97) / 97.f;
  EXPECT(ix->Train(train).ok() && ix->IsTrained());
  EXPECT(!ix->NeedToSave(20000));  // trained, no rows
  EXPECT(ix->Add(rows(ivf, 10, 1, 1)).ok() && ix->NeedToSave(20000));
  const Case hnsw{"hnsw_deleted", pb::common::VECTOR_INDEX_TYPE_HNSW, pb::common::METRIC_TYPE_L2, 16, 0, 0, 0, 10};
  auto h = make(hnsw);
  EXPECT(h->Add(rows(hnsw, 10, 1, 1)).ok());
  std::vector<int64_t> all;
  for (int64_t i = 1; i <= 10; ++i) all.push_back(i);
  EXPECT(h->Delete(all).ok());
  EXPECT(h->NeedToSave(20000));  // no live row, but deleted nodes: live + deleted != 0
  const Case fl{"flat_emptied", pb::common::VECTOR_INDEX_TYPE_FLAT, pb::common::METRIC_TYPE_L2, 16, 0, 0, 0, 10};
  auto f = make(fl);
  EXPECT(f->Add(rows(fl, 10, 1, 1)).ok() && f->Delete(all).ok());
  EXPECT(!f->NeedToSave(20000));
  VectorIndexB200::support_fork_save = false;
}

int main(int argc, char** argv) {
  const std::string dir = argc > 1 ? argv[1] : "/tmp";
  test_default_off(dir);
  using T = pb::common::VectorIndexType;
  const Case cases[] = {
      {"flat_l2", T::VECTOR_INDEX_TYPE_FLAT, pb::common::METRIC_TYPE_L2, 32, 0, 0, 0, 3000},
      {"flat_cosine", T::VECTOR_INDEX_TYPE_FLAT, pb::common::METRIC_TYPE_COSINE, 32, 0, 0, 0, 3000},
      {"ivf_flat_ip", T::VECTOR_INDEX_TYPE_IVF_FLAT, pb::common::METRIC_TYPE_INNER_PRODUCT, 32, 16, 0, 0, 3000},
      {"ivf_pq_inner_flat", T::VECTOR_INDEX_TYPE_IVF_PQ, pb::common::METRIC_TYPE_L2, 32, 16, 8, 8, 1000},
      {"ivf_pq", T::VECTOR_INDEX_TYPE_IVF_PQ, pb::common::METRIC_TYPE_L2, 32, 8, 8, 4, 5000},
      {"hnsw_l2", T::VECTOR_INDEX_TYPE_HNSW, pb::common::METRIC_TYPE_L2, 32, 0, 0, 0, 2000},
      {"binary_flat", T::VECTOR_INDEX_TYPE_BINARY_FLAT, pb::common::METRIC_TYPE_HAMMING, 64, 0, 0, 0, 3000},
      {"binary_ivf_flat", T::VECTOR_INDEX_TYPE_BINARY_IVF_FLAT, pb::common::METRIC_TYPE_HAMMING, 64, 16, 0, 0, 3000},
  };
  for (const Case& c : cases) test_case(c, dir);
  test_need_to_save_edges();
  printf(g_fail ? "PLUGIN SNAPSHOT TESTS FAILED: %d\n" : "PLUGIN SNAPSHOT TESTS OK%.0d\n", g_fail);
  return g_fail ? 1 : 0;
}
