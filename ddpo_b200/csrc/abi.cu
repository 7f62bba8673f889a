// Status handling, device queries and TMA tensor-map encoding for libddpo_b200.
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include "common.cuh"

namespace ddpo {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return DDPO_ERR_CUDA;
}

int num_sms() {
  static thread_local int cached_dev = -1;
  static thread_local int cached = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (dev != cached_dev) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    cached = n;
    cached_dev = dev;
  }
  return cached;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

int make_tensor_map(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides,
                    int swizzle_128b) {
  PFN_encodeTiled enc = get_encode();
  if (enc == nullptr) {
    set_error("cuTensorMapEncodeTiled driver entry point unavailable");
    return DDPO_ERR_CUDA;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    set_error("tensor map base %p not 16-byte aligned", base);
    return DDPO_ERR_INVALID;
  }
  cuuint64_t d[5], s[4];
  cuuint32_t b[5], e[5];
  for (int i = 0; i < rank; ++i) {
    d[i] = dims[i];
    b[i] = box[i];
    e[i] = elem_strides ? elem_strides[i] : 1;
    if (i + 1 < rank) {
      s[i] = strides_bytes[i];
      if (s[i] % 16 != 0) {
        set_error("tensor map stride %llu not a multiple of 16 bytes", (unsigned long long)s[i]);
        return DDPO_ERR_INVALID;
      }
    }
  }
  CUtensorMapDataType dt = elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = enc(out, dt, (cuuint32_t)rank, const_cast<void*>(base), d, s, b, e, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_128b == 1 ? CU_TENSOR_MAP_SWIZZLE_128B : swizzle_128b == 2 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed: %d (rank %d dims %llu,%llu,%llu,%llu box %u,%u,%u,%u)", (int)r, rank,
              (unsigned long long)d[0], (unsigned long long)(rank > 1 ? d[1] : 0),
              (unsigned long long)(rank > 2 ? d[2] : 0), (unsigned long long)(rank > 3 ? d[3] : 0), b[0],
              rank > 1 ? b[1] : 0, rank > 2 ? b[2] : 0, rank > 3 ? b[3] : 0);
    return DDPO_ERR_CUDA;
  }
  return DDPO_OK;
}

}  // namespace ddpo

extern "C" const char* ddpo_last_error(void) { return ddpo::g_err; }
extern "C" int ddpo_device_sm_count(void) {
  int n = ddpo::num_sms();
  if (n <= 0) {
    ddpo::set_error("no CUDA device");
    return DDPO_ERR_CUDA;
  }
  return n;
}
extern "C" int ddpo_abi_version(void) { return 3; }
