// Shared by the translation units of libmetis_b200.so (not part of the C ABI).
#ifndef METIS_INTERNAL_H
#define METIS_INTERNAL_H
#include <cuda_runtime.h>

#include <cstdint>

namespace metis {
// record the message returned by metis_last_error() and return METIS_E_CUDA / METIS_E_ARG
int fail_cuda(cudaError_t e, const char *what);
int fail_arg(const char *what);

// `v` rounded up to a multiple of 256 bytes: every piece of a workspace starts on such a boundary
inline int64_t align256(int64_t v) { return (v + 255) & ~(int64_t)255; }

// the first 256-byte boundary at or after `p`: where a caller's workspace is carved from
inline uint8_t *align_workspace(void *p) {
    return reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(p) + 255) & ~(uintptr_t)255);
}
}  // namespace metis
#endif
