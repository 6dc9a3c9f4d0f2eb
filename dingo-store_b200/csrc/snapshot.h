// snapshot.h — the index handle and its staged snapshot image, visible to host-only translation units.
//
// b200vs_save_stage builds, in the parent process, the exact bytes b200vs_save would write and keeps them in the handle;
// b200vs_save_staged (snapshot_write.cc) writes them from the child of a fork().  This header includes no CUDA header, so
// the child's side can be compiled without any.
#pragma once
#include <cstddef>
#include <cstdint>
#include <memory>
#include <string>

#include "../../include/b200vs.h"

namespace b200vs {

struct IndexBase;
extern thread_local std::string g_last_error;  // b200vs_last_error's text

// A snapshot file held in ordinary pageable heap memory, which a forked child inherits copy-on-write.  Page-locked or
// CUDA-registered host memory is not guaranteed to be mapped in such a child.
struct SnapshotImage {
  std::unique_ptr<uint8_t[]> bytes;
  size_t len = 0;
  void alloc(size_t n) { bytes.reset(new uint8_t[n > 0 ? n : 1]); len = n; }  // left uninitialised: every byte is written
  void reset() { bytes.reset(); len = 0; }
};

}  // namespace b200vs

struct b200vs_index {  // the opaque handle of include/b200vs.h
  b200vs::IndexBase* impl;
  b200vs::SnapshotImage image;  // b200vs_save_stage's image, none when bytes is null
};
