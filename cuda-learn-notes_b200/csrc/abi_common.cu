// Error reporting, device query and TMA tensor-map encoding for libb200k.so (see abi_common.cuh).
#include "abi_common.cuh"

#include <cstring>
#include <map>
#include <mutex>
#include <utility>

namespace b200k {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int get_device_info(DeviceInfo* out) {
  static std::mutex mu;
  static DeviceInfo cache[64];
  int dev = 0;
  B200K_CHECK_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return set_error(B200K_ECUDA, "device ordinal %d out of range", dev);
  std::lock_guard<std::mutex> lock(mu);
  DeviceInfo& c = cache[dev];
  if (c.device != dev) {
    DeviceInfo d;
    B200K_CHECK_CUDA(cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, dev));
    B200K_CHECK_CUDA(cudaDeviceGetAttribute(&d.cc_major, cudaDevAttrComputeCapabilityMajor, dev));
    B200K_CHECK_CUDA(cudaDeviceGetAttribute(&d.cc_minor, cudaDevAttrComputeCapabilityMinor, dev));
    B200K_CHECK_CUDA(cudaDeviceGetAttribute(&d.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    d.device = dev;
    c = d;
  }
  if (c.cc_major != 9 || c.cc_minor != 0)
    return set_error(B200K_EARCH, "libb200k needs a compute-capability 9.0 device (H100, sm_90a); device %d is %d.%d",
                     dev, c.cc_major, c.cc_minor);
  *out = c;
  return B200K_OK;
}

int ensure_dynamic_smem(const void* func, int device, int bytes) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, int> have;
  std::lock_guard<std::mutex> lock(mu);
  auto it = have.find({func, device});
  if (it != have.end() && it->second >= bytes) return B200K_OK;
  B200K_CHECK_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  have[{func, device}] = bytes;
  return B200K_OK;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int get_encode_fn(EncodeTiledFn* fn) {
  static EncodeTiledFn cached = nullptr;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  if (!cached) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &p, 12000, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p)
      return set_error(B200K_ECUDA, "cuTensorMapEncodeTiled not available from the driver (%s)",
                       cudaGetErrorString(e));
    cached = reinterpret_cast<EncodeTiledFn>(p);
  }
  *fn = cached;
  return B200K_OK;
}

int make_tmap(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims, const uint64_t* strides,
              const uint32_t* box) {
  EncodeTiledFn fn;
  int rc = get_encode_fn(&fn);
  if (rc) return rc;
  bool aligned = (reinterpret_cast<uintptr_t>(base) & 15) == 0;
  for (int i = 0; i < rank - 1; ++i) aligned = aligned && (strides[i] & 15) == 0;
  if (!aligned)
    return set_error(B200K_EALIGN, "TMA needs a 16-byte aligned base (%p) and strides (row stride %llu bytes)", base,
                     (unsigned long long)strides[0]);
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUtensorMapDataType type = elem_bytes == 4   ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                   : elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                                     : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUresult r = fn(out, type, rank,
                  const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(B200K_ECUDA,
                     "cuTensorMapEncodeTiled(%d-byte elements, dims %llu x %llu x %llu, box %u x %u x %u, innermost first) "
                     "failed with CUresult %d",
                     elem_bytes, (unsigned long long)dims[0], (unsigned long long)dims[1],
                     (unsigned long long)(rank == 3 ? dims[2] : 1), box[0], box[1], rank == 3 ? box[2] : 1u, (int)r);
  return B200K_OK;
}

}  // namespace b200k

extern "C" {
int b200k_abi_version(void) { return B200K_ABI_VERSION; }
const char* b200k_last_error(void) { return b200k::g_err; }
int b200k_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  b200k::DeviceInfo d;
  int rc = b200k::get_device_info(&d);
  if (rc) return rc;
  if (sm_count) *sm_count = d.sm_count;
  if (cc_major) *cc_major = d.cc_major;
  if (cc_minor) *cc_minor = d.cc_minor;
  return B200K_OK;
}
}
