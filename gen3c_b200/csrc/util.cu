// Host-side utilities shared by all translation units of libgen3c_b200.so:
// thread-local error string, CUDA error mapping, TMA descriptor encoding through the driver
// entry point (no link-time dependency on libcuda).
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>

#include "common.cuh"

namespace g3c {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  set_error("CUDA error %d (%s) at %s:%d in `%s`", (int)e, cudaGetErrorString(e), file, line, what);
  return G3C_ECUDA;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (PFN_encodeTiled)p;
  });
  return fn;
}

int make_tmap_bf16_sw128(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                         const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapDataType dtype) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return G3C_ECUDA;
  }
  if (rank < 2 || rank > 4) {
    set_error("tensor map rank %d unsupported", rank);
    return G3C_EINVAL;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    set_error("TMA base pointer %p not 16-byte aligned", base);
    return G3C_EINVAL;
  }
  cuuint64_t gdims[4];
  cuuint64_t gstr[3];
  cuuint32_t gbox[4], estr[4];
  for (int i = 0; i < rank; ++i) {
    gdims[i] = dims[i];
    gbox[i] = box[i];
    estr[i] = 1;
  }
  for (int i = 0; i < rank - 1; ++i) {
    gstr[i] = strides_bytes[i];
    if (gstr[i] % 16 != 0) {
      set_error("TMA stride %llu (dim %d) not a multiple of 16 bytes",
                (unsigned long long)gstr[i], i + 1);
      return G3C_EINVAL;
    }
  }
  CUresult r = enc(out, dtype, (cuuint32_t)rank, const_cast<void*>(base),
                   gdims, gstr, gbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu box %u,%u)",
              (int)r, rank, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0],
              box[1]);
    return G3C_ECUDA;
  }
  return G3C_OK;
}

int make_tmap_f32_sw128(CUtensorMap* out, const void* base, const uint64_t* dims,
                        const uint64_t* strides_bytes, const uint32_t* box) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return G3C_ECUDA;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || strides_bytes[0] % 16 != 0) {
    set_error("TMA f32 map: base %p / stride %llu not 16-byte aligned", base,
              (unsigned long long)strides_bytes[0]);
    return G3C_EINVAL;
  }
  cuuint64_t gdims[2] = {dims[0], dims[1]};
  cuuint64_t gstr[1] = {strides_bytes[0]};
  cuuint32_t gbox[2] = {box[0], box[1]}, estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdims, gstr, gbox, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(f32) failed with CUresult %d", (int)r);
    return G3C_ECUDA;
  }
  return G3C_OK;
}

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n = 132;
  }
  return n;
}

}  // namespace g3c

extern "C" {

const char* g3c_last_error(void) { return g3c::g_err; }

int g3c_version(void) { return 100; }

int g3c_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  G3C_CUDA(cudaGetDevice(&dev));
  int a = 0, b = 0, c = 0;
  G3C_CUDA(cudaDeviceGetAttribute(&a, cudaDevAttrMultiProcessorCount, dev));
  G3C_CUDA(cudaDeviceGetAttribute(&b, cudaDevAttrComputeCapabilityMajor, dev));
  G3C_CUDA(cudaDeviceGetAttribute(&c, cudaDevAttrComputeCapabilityMinor, dev));
  if (sm_count) *sm_count = a;
  if (cc_major) *cc_major = b;
  if (cc_minor) *cc_minor = c;
  return G3C_OK;
}

}  // extern "C"
