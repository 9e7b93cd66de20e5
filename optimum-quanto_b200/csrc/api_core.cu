// The host-side state every translation unit shares (last-error text, per-device caches, TMA descriptor encoding, test
// hooks, developer flags) and the extern "C" entry points that query or set it (include/quanto_b200.h).
#include "../../include/quanto_b200.h"

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>

#include "host_common.cuh"

namespace qb {

static thread_local char g_err[512] = "";
static thread_local int g_family = 0;
static std::atomic<int> g_override[OVR_COUNT];
#ifdef QB_DEVELOPER_KNOCKOUTS
static std::atomic<int> g_dbg{0};
static std::atomic<long long*> g_trace{nullptr};
#endif

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return OK;
  return fail(ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

void set_kernel_family(int family) { g_family = family; }

int test_override(int key) { return (key >= 0 && key < OVR_COUNT) ? g_override[key].load(std::memory_order_relaxed) : 0; }

int debug_flags() {
#ifdef QB_DEVELOPER_KNOCKOUTS
  return g_dbg.load(std::memory_order_relaxed);
#else
  return 0;
#endif
}
long long* debug_trace() {
#ifdef QB_DEVELOPER_KNOCKOUTS
  return g_trace.load(std::memory_order_relaxed);
#else
  return nullptr;
#endif
}

// ---------------------------------------------------------------------------------------------
// per-device caches
// ---------------------------------------------------------------------------------------------
int current_device() {
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  return dev;
}

struct DeviceFacts {
  std::atomic<int> sms{0};
  std::atomic<int> cc_major{-1};
};
static DeviceFacts g_dev[kMaxDevices];

int current_sm_count() {
  const int dev = current_device();
  if (dev < 0) return kNumSMsH100;
  if (dev < kMaxDevices) {
    const int cached = g_dev[dev].sms.load(std::memory_order_relaxed);
    if (cached > 0) return cached;
  }
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (sms <= 0) sms = kNumSMsH100;
  if (dev < kMaxDevices) g_dev[dev].sms.store(sms, std::memory_order_relaxed);
  return sms;
}

int check_arch(const char* what) {
  int dev = -1;
  const cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return fail(ERR_CUDA, "%s: no current CUDA device: %s", what, cudaGetErrorString(e));
  int major = (dev < kMaxDevices) ? g_dev[dev].cc_major.load(std::memory_order_relaxed) : -1;
  if (major < 0) {
    major = 0;
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    if (dev < kMaxDevices) g_dev[dev].cc_major.store(major, std::memory_order_relaxed);
  }
  if (major == 9) return OK;
  return fail(ERR_ARCH, "%s: quanto_b200 kernels are built for sm_90a only (device %d is sm_%d)", what, dev, major);
}

// ---------------------------------------------------------------------------------------------
// driver entry point for cuTensorMapEncodeTiled (no link-time dependency on libcuda)
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static int encode_2d(CUtensorMap* map, const void* base, int dt, int64_t rows, int64_t cols, int64_t pitch_elems,
                     int box_cols, int box_rows, CUtensorMapSwizzle swz) {
  EncodeTiledFn enc = get_encode_fn();
  if (enc == nullptr) return fail(ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  CUtensorMapDataType type;
  int esz;
  switch (dt) {
    case DT_BF16: type = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16; esz = 2; break;
    case DT_F16: type = CU_TENSOR_MAP_DATA_TYPE_FLOAT16; esz = 2; break;
    case DT_F32: type = CU_TENSOR_MAP_DATA_TYPE_FLOAT32; esz = 4; break;
    default: type = CU_TENSOR_MAP_DATA_TYPE_UINT8; esz = 1; break;
  }
  if (!aligned16(base)) return fail(ERR_ARG, "TMA operand not 16-byte aligned");
  if ((pitch_elems * esz) % 16 != 0)
    return fail(ERR_ARG, "TMA row pitch %lld not a multiple of 16 bytes", (long long)(pitch_elems * esz));
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(pitch_elems) * esz};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t estride[2] = {1, 1};
  CUresult r = enc(map, type, 2, const_cast<void*>(base), gdim, gstride, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", static_cast<int>(r));
  return OK;
}

int make_tmap_2d(CUtensorMap* map, const void* base, int dt, int64_t rows, int64_t cols, int box_rows) {
  const int esz = dtype_size(dt);
  return encode_2d(map, base, dt, rows, cols, cols, 128 / esz, box_rows, CU_TENSOR_MAP_SWIZZLE_128B);
}

int make_tmap_planes(CUtensorMap* map, const void* base, int dt, int64_t rows, int64_t cols, int box_rows) {
  EncodeTiledFn enc = get_encode_fn();
  if (enc == nullptr) return fail(ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  if (dt != DT_BF16 && dt != DT_F16) return fail(ERR_ARG, "plane tensor map: 16-bit elements only");
  if (!aligned16(base)) return fail(ERR_ARG, "TMA operand not 16-byte aligned");
  if (cols % 16 != 0) return fail(ERR_ARG, "plane tensor map: cols %lld not a multiple of 16", (long long)cols);
  const CUtensorMapDataType type = dt == DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const cuuint64_t half = static_cast<cuuint64_t>(cols / 2);
  const cuuint64_t gdim[3] = {half, 2, static_cast<cuuint64_t>(rows)};
  const cuuint64_t gstride[2] = {half * 2, static_cast<cuuint64_t>(cols) * 2};
  const cuuint32_t box[3] = {64, 1, static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t estride[3] = {1, 1, 1};
  CUresult r = enc(map, type, 3, const_cast<void*>(base), gdim, gstride, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(ERR_CUDA, "cuTensorMapEncodeTiled (planes) failed with CUresult %d", static_cast<int>(r));
  return OK;
}

int make_tmap_packed(CUtensorMap* map, const uint8_t* packed, int64_t rows, int64_t cols, int box_rows) {
  return encode_2d(map, packed, DT_U8, rows, cols, cols, 64, box_rows, CU_TENSOR_MAP_SWIZZLE_64B);
}

int make_tmap_3d_bytes(CUtensorMap* map, const void* base, int64_t batch, int64_t rows, int64_t cols,
                       int64_t batch_stride, int box_rows) {
  EncodeTiledFn enc = get_encode_fn();
  if (enc == nullptr) return fail(ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  if (!aligned16(base)) return fail(ERR_ARG, "TMA operand not 16-byte aligned");
  if (cols % 16 != 0 || batch_stride % 16 != 0)
    return fail(ERR_ARG, "TMA row pitch %lld / batch stride %lld not a multiple of 16 bytes", (long long)cols,
                (long long)batch_stride);
  const cuuint64_t gdim[3] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(batch)};
  const cuuint64_t gstride[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(batch_stride)};
  const cuuint32_t box[3] = {128, static_cast<cuuint32_t>(box_rows), 1};
  const cuuint32_t estride[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), gdim, gstride, box, estride,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(ERR_CUDA, "cuTensorMapEncodeTiled (3-d) failed with CUresult %d", static_cast<int>(r));
  return OK;
}

}  // namespace qb

using namespace qb;

extern "C" {

int qb200_version(void) { return 200; }

int qb200_device_supported(int device) {
  int major = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device) != cudaSuccess) return -1;
  return major == 9 ? 1 : 0;
}

const char* qb200_last_error(void) { return g_err; }
int qb200_last_kernel_family(void) { return g_family; }

int qb200_test_override(int key, int value) {
  if (key < 0 || key >= OVR_COUNT) return fail(ERR_ARG, "test_override: unknown key %d", key);
  g_override[key].store(value, std::memory_order_relaxed);
  return OK;
}

void qb200_debug_set_trace(void* device_buffer) {
#ifdef QB_DEVELOPER_KNOCKOUTS
  g_trace.store(static_cast<long long*>(device_buffer));
#else
  (void)device_buffer;
#endif
}
void qb200_debug_set_flags(int flags) {
#ifdef QB_DEVELOPER_KNOCKOUTS
  g_dbg.store(flags);
#else
  (void)flags;
#endif
}
int qb200_debug_flags(void) { return debug_flags(); }
int qb200_developer_build(void) {
#ifdef QB_DEVELOPER_KNOCKOUTS
  return 1;
#else
  return 0;
#endif
}

}  // extern "C"
