// Host-side plumbing shared by the translation units that hold the extern "C" entry points: status reporting,
// per-DEVICE caches (SM count, architecture check, dynamic shared-memory opt-in), the persistent-kernel launch, TMA
// descriptor encoding, the mapping of run-time dtype codes to kernel template arguments and the test hooks that pick
// among equivalent kernels.
#pragma once

#include <atomic>
#include <cstdint>
#include <type_traits>

#include "common.cuh"

namespace qb {

// ---- status (defined in api_core.cu; the message is thread-local, read back through qb200_last_error) ----------
int fail(int code, const char* fmt, ...);
// OK, or ERR_CUDA with the message "<what>: <the runtime's reason>".  Launchers pass cudaGetLastError() straight in:
// that call clears a non-sticky error, so a later call could no longer report it.
int check_cuda(cudaError_t e, const char* what);
void set_kernel_family(int family);

// ---- per-device facts.  cudaFuncSetAttribute, the SM count and the compute capability belong to a DEVICE, not to the
// process: a process that drives several GPUs (device_map="auto", pipeline stages) calls the same entry points under
// different current devices, so everything below is keyed by cudaGetDevice().
constexpr int kMaxDevices = 64;
int current_device();       // cudaGetDevice, -1 on error
int current_sm_count();     // multiprocessors of the current device
int check_arch(const char* what);  // OK when the current device is sm_90 (Hopper), else ERR_ARCH / ERR_CUDA

// Opt the kernel into `bytes` of dynamic shared memory on the current device (once per kernel and device).  The kernel
// is a template ARGUMENT: one static per kernel function (kernels of different configurations share a pointer TYPE).
template <auto kernel>
int ensure_dyn_smem(int bytes) {
  static std::atomic<uint64_t> done{0};  // one bit per device
  const int dev = current_device();
  if (dev < 0) return fail(ERR_CUDA, "no current CUDA device");
  if (dev < kMaxDevices && (done.load(std::memory_order_acquire) >> dev) & 1ull) return OK;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute(MaxDynamicSharedMemorySize)");
  // the whole unified L1 / shared-memory array as shared memory: a kernel that asks for ~110 KB must be able to run two
  // CTAs per SM (the driver otherwise picks the smallest carve-out that holds ONE of them)
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute(PreferredSharedMemoryCarveout)");
  if (dev < kMaxDevices) done.fetch_or(1ull << dev, std::memory_order_release);
  return OK;
}

// Launch with the programmatic-stream-serialization attribute (PDL, see common.cuh) when `pdl`, else an ordinary launch.
template <class... KArgs, class... Args>
cudaError_t launch_kernel_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl,
                              Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Launch a persistent wgmma kernel (wgmma_pipe.cuh): one CTA per SM, or per tile when there are fewer tiles.  Layout is
// the kernel's PipeLayout, which fixes its block size and dynamic shared memory.
template <auto kernel, class Layout, class... Args>
int launch_persistent(int tiles, cudaStream_t stream, const char* what, const Args&... args) {
  int rc = ensure_dyn_smem<kernel>(Layout::SMEM_BYTES);
  if (rc != OK) return rc;
  const int grid = tiles < current_sm_count() ? tiles : current_sm_count();
  kernel<<<grid, Layout::NTHREADS, Layout::SMEM_BYTES, stream>>>(args...);
  return check_cuda(cudaGetLastError(), what);
}

// Row-major [rows, cols] matrix of `dt` elements; box = 128 bytes of a row x box_rows rows, 128-byte swizzle.
int make_tmap_2d(CUtensorMap* map, const void* base, int dt, int64_t rows, int64_t cols, int box_rows);
// Row-major [rows, cols] 16-bit matrix described as [rows, 2, cols/2] (two column planes); box = 64 elements of one
// plane x box_rows rows, 128-byte swizzle.  A box never crosses cols/2: past the end of a plane TMA fills zeros.
int make_tmap_planes(CUtensorMap* map, const void* base, int dt, int64_t rows, int64_t cols, int box_rows);
// Packed int4 weights [rows, cols] bytes; box = 64 bytes of a row x box_rows rows, 64-byte swizzle (16-byte chunk s of
// row r at chunk s ^ ((r >> 1) & 3)).
int make_tmap_packed(CUtensorMap* map, const uint8_t* packed, int64_t rows, int64_t cols, int box_rows);
// [batch, rows, cols] bytes, rows dense (pitch = cols), batches `batch_stride` bytes apart; box = 128 bytes of a row x
// box_rows rows of one batch, 128-byte swizzle.  A box never crosses a batch: past `rows` TMA fills zeros.
int make_tmap_3d_bytes(CUtensorMap* map, const void* base, int64_t batch, int64_t rows, int64_t cols,
                       int64_t batch_stride, int box_rows);

// TMA operands, vector loads and bulk copies need 16-byte aligned addresses
inline bool aligned16(const void* ptr) { return reinterpret_cast<uintptr_t>(ptr) % 16 == 0; }

// Grid of a grid-stride kernel: one CTA per `per_cta` work items, at least 1 and at most `ctas_per_sm` CTAs for each SM
// of a 132-SM H100 SXM.
inline int capped_grid(int64_t items, int64_t per_cta, int ctas_per_sm) {
  const int64_t blocks = (items + per_cta - 1) / per_cta;
  const int64_t cap = static_cast<int64_t>(kNumSMsH100) * ctas_per_sm;
  return static_cast<int>(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

inline bool is_float_dtype(int dt) { return dt == DT_F32 || dt == DT_F16 || dt == DT_BF16; }
inline bool is_code_dtype(int dt) { return dt == DT_I8 || dt == DT_E4M3 || dt == DT_E5M2 || dt == DT_E4M3FNUZ; }

// Lanes of the team that owns one grouped row of `group` elements (8 per lane): group / 8 rounded up to a power of two
inline int team_lanes(int group) {
  int tl = 1;
  while (tl < group / 8) tl <<= 1;
  return tl;
}

// ---- run-time codes -> template arguments.  Each dispatch_* helper calls the generic lambda `f` with a tag type for the
// code it is given, so that `f` names the kernel configuration once and instantiates it for exactly the codes listed
// here.  The entry points validate their arguments first: a code outside a helper's set is a dispatch bug, reported as
// ERR_ARG rather than run as some other type.

// 16-bit activation dtype: the staged element type and the MMA kind that consumes it
template <typename WT_, MmaKind KIND_>
struct Act16 {
  using WT = WT_;
  static constexpr MmaKind KIND = KIND_;
};

// DT_BF16 / DT_F16 -> Act16<__nv_bfloat16, BF16> / Act16<__half, F16>
template <class F>
int dispatch_act16(int dtype, F&& f) {
  if (dtype == DT_BF16) return f(Act16<__nv_bfloat16, MmaKind::BF16>{});
  if (dtype == DT_F16) return f(Act16<__half, MmaKind::F16>{});
  return fail(ERR_ARG, "dispatch: activation dtype %d is neither bf16 nor fp16", dtype);
}

// shift_is_int -> std::bool_constant ZP: the int4 shift is an integer zero-point (else a float shift)
template <class F>
int dispatch_zp(int shift_is_int, F&& f) {
  if (shift_is_int != 0) return f(std::true_type{});
  return f(std::false_type{});
}

// the dtype x zero-point pair of the int4 kernels: f(Act16 tag, bool_constant ZP)
template <class F>
int dispatch_act16_zp(int dtype, int shift_is_int, F&& f) {
  return dispatch_act16(dtype, [&](auto act) { return dispatch_zp(shift_is_int, [&](auto zp) { return f(act, zp); }); });
}

// 8-bit weight dtype -> std::integral_constant WKIND: 0 int8, 1 float8_e4m3fn, 2 float8_e5m2, 3 float8_e4m3fnuz
template <class F>
int dispatch_wkind(int w_dtype, F&& f) {
  switch (w_dtype) {
    case DT_I8: return f(std::integral_constant<int, 0>{});
    case DT_E4M3: return f(std::integral_constant<int, 1>{});
    case DT_E5M2: return f(std::integral_constant<int, 2>{});
    case DT_E4M3FNUZ: return f(std::integral_constant<int, 3>{});
    default: return fail(ERR_ARG, "dispatch: weight dtype %d is not an 8-bit type", w_dtype);
  }
}

// rows per wgmma tile 64 / 128 -> std::integral_constant MWG (consumer warpgroups) 1 / 2
template <class F>
int dispatch_mwg(int tile_m, F&& f) {
  if (tile_m == 64) return f(std::integral_constant<int, 1>{});
  if (tile_m == 128) return f(std::integral_constant<int, 2>{});
  return fail(ERR_ARG, "dispatch: tile height %d is neither 64 nor 128", tile_m);
}

// float element dtype: the element type T
template <typename T_>
struct Float {
  using T = T_;
};

// DT_F32 / DT_F16 / DT_BF16 -> Float<float> / Float<__half> / Float<__nv_bfloat16>
template <class F>
int dispatch_float(int dtype, F&& f) {
  switch (dtype) {
    case DT_F32: return f(Float<float>{});
    case DT_F16: return f(Float<__half>{});
    case DT_BF16: return f(Float<__nv_bfloat16>{});
    default: return fail(ERR_ARG, "dispatch: dtype %d is not a float type", dtype);
  }
}

// 8-bit code dtype -> std::integral_constant<int, DT_*>
template <class F>
int dispatch_code8(int dtype, F&& f) {
  switch (dtype) {
    case DT_I8: return f(std::integral_constant<int, DT_I8>{});
    case DT_E4M3: return f(std::integral_constant<int, DT_E4M3>{});
    case DT_E5M2: return f(std::integral_constant<int, DT_E5M2>{});
    case DT_E4M3FNUZ: return f(std::integral_constant<int, DT_E4M3FNUZ>{});
    default: return fail(ERR_ARG, "dispatch: dtype %d is not an 8-bit code type", dtype);
  }
}

// bits per packed weight 2 / 4 -> std::integral_constant BITS
template <class F>
int dispatch_bits(int bits, F&& f) {
  if (bits == 4) return f(std::integral_constant<int, 4>{});
  if (bits == 2) return f(std::integral_constant<int, 2>{});
  return fail(ERR_ARG, "dispatch: bits %d is neither 2 nor 4", bits);
}

// group (a multiple of 8, at most 256) -> std::integral_constant TL = team_lanes(group) in 1 ... 32
template <class F>
int dispatch_team_lanes(int group, F&& f) {
  switch (team_lanes(group)) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 8: return f(std::integral_constant<int, 8>{});
    case 16: return f(std::integral_constant<int, 16>{});
    case 32: return f(std::integral_constant<int, 32>{});
    default: return fail(ERR_ARG, "dispatch: group %d needs more than 32 lanes", group);
  }
}

// ---- test hooks (include/quanto_b200.h: qb200_test_override).  Every value selects a kernel that computes the same
// result; 0 = automatic choice.  They exist so that the test-suite can execute every shipped instantiation.
enum : int { OVR_TILE_M = 0 /* 64 | 128 rows per wgmma tile; 256: the int4 swap-AB kernel at 256 tokens */, OVR_QBYTES_TILE_N = 1 /* int8: 128 | 256 */,
             OVR_INT4_ROUTE = 2, OVR_QBYTES_ROUTE = 3, OVR_GEMV_PRODUCER = 4,
             OVR_PDL = 5 /* 1 = no programmatic dependent launch */,
             OVR_GEMV_SHAPE = 6 /* 2 = the two-CTAs-per-SM shape of the ring gemv (M <= 2) */,
             OVR_INT4_EPILOGUE = 7 /* 1 = the int4 wgmma epilogue stores without TMA */,
             OVR_BMM_ROUTE = 8 /* qbytes_bmm: 2 = CUDA-core kernel, 3 = K-major copy of B + wgmma for any B layout */,
             OVR_CONV_TILE_M = 9 /* conv2d: 64 | 128 rows (output pixels) per tile */,
             OVR_COUNT = 10 };
// OVR_INT4_ROUTE values
enum : int { ROUTE_AUTO = 0, ROUTE_INT4_GENERAL = 1, ROUTE_INT4_GEMV = 3, ROUTE_INT4_RING = 4, ROUTE_INT4_RING2 = 8 };
// OVR_QBYTES_ROUTE values
enum : int { ROUTE_QBYTES_SIMT = 2 };
// OVR_BMM_ROUTE values
enum : int { ROUTE_BMM_SIMT = 2, ROUTE_BMM_TRANSPOSE = 3 };
int test_override(int key);

// Rows per wgmma tile: one consumer warpgroup (64 rows) while M <= 64, so that small batches do not pay for empty MMA
// rows, else 128; test override OVR_TILE_M forces either.
inline int wgmma_tile_m(int64_t m) {
  int tile_m = m <= 64 ? 64 : 128;
  const int force_m = test_override(OVR_TILE_M);
  if (force_m == 64 || force_m == 128) tile_m = force_m;
  return tile_m;
}

// log2(group) when group is a power of two, else -1
inline int group_log2(int group) {
  for (int b = 0; b < 31; ++b)
    if ((1 << b) == group) return b;
  return -1;
}

// ---- developer knock-outs: only a KNOCKOUTS=1 build honours them; a release build reports and uses 0
int debug_flags();
long long* debug_trace();

}  // namespace qb
