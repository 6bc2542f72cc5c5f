// Host-side helpers shared by every translation unit behind the C ABI (include/b200k.h):
// error reporting, driver-entry-point lookup for cuTensorMapEncodeTiled (so the library has no link-time
// dependency on libcuda.so and can be dlopen'ed on a GPU-less box), device properties cache.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdint>
#include <cstdio>

#include "../../include/b200k.h"

namespace b200k {

int set_error(int code, const char* fmt, ...);  // returns `code`
#define B200K_CHECK_CUDA(expr)                                                                      \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess)                                                                          \
      return ::b200k::set_error(B200K_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                                __FILE__, __LINE__);                                                \
  } while (0)

struct DeviceInfo {
  int device = -1;
  int sm_count = 0;
  int cc_major = 0, cc_minor = 0;
  int max_smem_optin = 0;
};
// Properties of the current device; fails (B200K_EARCH) unless it is compute capability 9.0.
int get_device_info(DeviceInfo* out);

// cudaFuncAttributeMaxDynamicSharedMemorySize is per function and per device.  One mutex-protected table for every
// launcher in the library; a (function, device) pair is recorded only after the attribute call succeeded, and the
// recorded size only grows, so a transient failure is retried by the next launch instead of poisoning it.
int ensure_dynamic_smem(const void* func, int device, int bytes);

// TMA tensor map with 128-byte swizzle over a rank-2 or rank-3 global array of 2-byte elements (f16 and bf16 alike,
// encoded as FLOAT16) or 4-byte fp32 ones.  dims[rank] and box[rank] list the innermost dimension first; strides[rank - 1]
// are the byte strides of dims[1 ..].  The base and every stride must be multiples of 16 bytes (B200K_EALIGN otherwise).
int make_tmap(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims, const uint64_t* strides,
              const uint32_t* box);

}  // namespace b200k
