// Context object behind the opaque xivo_ctx handle + a small RAII device buffer.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

struct xivo_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
};

namespace xb {
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  bool failed = false;
  DevBuf() {}
  explicit DevBuf(size_t count) { alloc(count); }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
  // releases what it held; on failure the buffer is left empty
  bool alloc(size_t count) {
    release();
    failed = count && cudaMalloc(reinterpret_cast<void**>(&p), count * sizeof(T)) != cudaSuccess;
    if (failed) p = nullptr;
    else n = count;
    return !failed;
  }
  bool ok() const { return !failed; }
};
}  // namespace xb
