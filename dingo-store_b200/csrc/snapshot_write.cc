// snapshot_write.cc — b200vs_save_staged: write the image b200vs_save_stage staged in the handle to a file.
//
// The call is made from the child of a fork() of a multi-threaded process that owns a CUDA context (the snapshot path of
// VectorIndexSnapshotManager: LockWrite, fork, Save in the child, UnlockWrite in the parent).  Such a child cannot use the
// parent's CUDA context, and any lock another parent thread held at the fork stays held in the child forever.  So this
// translation unit is compiled by the host compiler without CUDA headers and cannot reach the CUDA runtime or driver
// (tests/test_snapshot_abi.py lists its undefined symbols), takes no library lock, logs nothing and starts no thread.
// The only library state it touches is the handle's image and the thread-local error text.
#include <fcntl.h>
#include <unistd.h>

#include <algorithm>
#include <cerrno>
#include <cstring>

#include "snapshot.h"

namespace {

int refuse(int code, const char* what, const char* path = nullptr, int err = 0) {
  try {
    b200vs::g_last_error = what;
    if (path) b200vs::g_last_error += std::string(" ") + path;
    if (err) b200vs::g_last_error += std::string(": ") + strerror(err);
  } catch (...) {
  }
  return code;
}

}  // namespace

extern "C" int b200vs_save_staged(b200vs_index* h, const char* path) {
  if (!h || !h->image.bytes) return refuse(B200VS_EILLEGAL_PARAMETERS, "no staged snapshot image (b200vs_save_stage)");
  if (!path || !*path) return refuse(B200VS_EILLEGAL_PARAMETERS, "path is empty");
  const int fd = open(path, O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0666);  // fopen(path, "wb")'s file
  if (fd < 0) return refuse(B200VS_EINTERNAL, "cannot open", path, errno);
  const uint8_t* p = h->image.bytes.get();
  size_t left = h->image.len;
  while (left > 0) {
    const ssize_t w = write(fd, p, std::min<size_t>(left, (size_t)1 << 30));
    if (w < 0 && errno == EINTR) continue;
    if (w <= 0) {
      const int err = w < 0 ? errno : EIO;
      close(fd);
      return refuse(B200VS_EINTERNAL, "short write to", path, err);
    }
    p += w;
    left -= (size_t)w;
  }
  // EINTR from close leaves the descriptor closed on Linux, and the data was already handed to the kernel
  if (close(fd) != 0 && errno != EINTR) return refuse(B200VS_EINTERNAL, "cannot close", path, errno);
  return B200VS_OK;
}
