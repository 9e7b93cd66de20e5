"""ctypes binding of the C-ABI library (include/quanto_b200.h).

The library is built in-tree by `__graft_entry__.build()` / `make -C optimum-quanto_b200/csrc` into
`quanto_b200/lib/libquanto_b200.so`.  There is no fallback: if the library is missing or a call fails the
caller gets an exception, never a silent CPU/eager path.

Role in the reference: replaces the lazy JIT pybind loader `optimum/quanto/library/extensions/extension.py:13-54`.
"""
import ctypes
import os
import threading

import torch

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libquanto_b200.so")

F32, F16, BF16, I8, U8, E4M3, E5M2, E4M3FNUZ = range(8)

DTYPE_CODE = {
    torch.float32: F32,
    torch.float16: F16,
    torch.bfloat16: BF16,
    torch.int8: I8,
    torch.uint8: U8,
    torch.float8_e4m3fn: E4M3,
    torch.float8_e5m2: E5M2,
    torch.float8_e4m3fnuz: E4M3FNUZ,
}

ERR_NAMES = {1: "invalid argument", 2: "unsupported configuration", 3: "CUDA error", 4: "unsupported architecture"}

EXPORTS = (
    "qb200_version",
    "qb200_device_supported",
    "qb200_last_error",
    "qb200_unpack",
    "qb200_quantize_symmetric",
    "qb200_dequantize_qbits",
    "qb200_qbits_mm",
    "qb200_qbits_mm_gather",
    "qb200_qbits_mm_workspace_bytes",
    "qb200_qbytes_mm",
    "qb200_qbytes_mm_quantized",
    "qb200_quantize_affine",
    "qb200_pack",
    "qb200_quantize_qbits_max",
    "qb200_absmax",
    "qb200_quantize_qbytes_absmax",
    "qb200_last_kernel_family",
    "qb200_debug_set_trace",
    "qb200_debug_set_flags",
    "qb200_debug_flags",
    "qb200_developer_build",
    "qb200_test_override",
    "qb200_qbits_ring_plan",
    "qb200_qbits_mm_grad_input",
    "qb200_qbytes_mm_grad_input",
    "qb200_quantize_qbits_hqq",
    "qb200_quantize_qbits_hqq_workspace_bytes",
    "qb200_hqq_shrink",
    "qb200_qbytes_bmm",
    "qb200_qbytes_bmm_workspace_bytes",
    "qb200_qbytes_softmax",
    "qb200_qbits_conv2d",
    "qb200_qbytes_conv2d",
    "qb200_layer_norm",
    "qb200_absmax_update",
)

# qb200_test_override keys (include/quanto_b200.h)
(OVR_TILE_M, OVR_QBYTES_TILE_N, OVR_INT4_ROUTE, OVR_QBYTES_ROUTE, OVR_GEMV_PRODUCER, OVR_PDL, OVR_GEMV_SHAPE,
 OVR_INT4_EPILOGUE, OVR_BMM_ROUTE, OVR_CONV_TILE_M) = range(10)
ROUTE_INT4_GENERAL, ROUTE_INT4_GEMV, ROUTE_INT4_RING, ROUTE_INT4_RING2 = 1, 3, 4, 8
ROUTE_QBYTES_SIMT = 2
ROUTE_BMM_SIMT, ROUTE_BMM_TRANSPOSE = 2, 3
GATHER_WAIT_INPUT, GATHER_WAIT_OUTPUT = 1, 2


class NativeLibraryError(RuntimeError):
    pass


class UnsupportedConfiguration(NativeLibraryError):
    """Raised for status QB200_ERR_UNSUPPORTED: the caller may compose other native kernels instead."""


_lib = None
_lock = threading.Lock()


def lib_path() -> str:
    return _LIB_PATH


def use_developer_library():
    """Developer tools only (tools/trace_*.py): load the `make KNOCKOUTS=1` build (timelines, knock-out flags) instead of the
    release library.  Must be called before the first load(); nothing in the package or in bench.py / tests calls it."""
    global _LIB_PATH
    if _lib is not None:
        raise NativeLibraryError("the native library is already loaded")
    _LIB_PATH = os.path.join(os.path.dirname(_LIB_PATH), "libquanto_b200_dev.so")


def load():
    """Load (once) and return the ctypes handle.  Raises NativeLibraryError when the .so is absent."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(_LIB_PATH):
            raise NativeLibraryError(
                f"{_LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C optimum-quanto_b200/csrc`). quanto_b200 has no CPU or eager fallback."
            )
        lib = ctypes.CDLL(_LIB_PATH)
        vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
        lib.qb200_version.restype = i32
        lib.qb200_device_supported.argtypes = [i32]
        lib.qb200_last_error.restype = ctypes.c_char_p
        lib.qb200_last_kernel_family.restype = i32
        lib.qb200_unpack.argtypes = [vp, vp, i64, i32, vp]
        lib.qb200_quantize_symmetric.argtypes = [vp, vp, vp, i64, i64, i32, i32, i32, vp]
        lib.qb200_dequantize_qbits.argtypes = [vp, vp, vp, vp, i64, i64, i32, i32, i32, i32, vp]
        lib.qb200_qbits_mm.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i32, i32, i32, i32, vp, i64, vp]
        lib.qb200_qbits_mm_gather.argtypes = [vp, vp, vp, vp, vp, ctypes.POINTER(vp), ctypes.POINTER(vp), i32, i32, i32,
                                              i64, i64, i64, i32, i32, i32, vp, i64, vp]
        lib.qb200_qbits_mm_workspace_bytes.argtypes = [i64, i64, i64]
        lib.qb200_qbits_mm_workspace_bytes.restype = i64
        lib.qb200_qbits_ring_plan.argtypes = [i64, i64, i64, i32, i32, i32, ctypes.POINTER(i32)]
        lib.qb200_qbits_ring_plan.restype = i32
        lib.qb200_debug_set_trace.argtypes = [vp]
        lib.qb200_debug_set_trace.restype = None
        lib.qb200_debug_set_flags.argtypes = [i32]
        lib.qb200_debug_set_flags.restype = None
        lib.qb200_debug_flags.restype = i32
        lib.qb200_developer_build.restype = i32
        lib.qb200_test_override.argtypes = [i32, i32]
        lib.qb200_qbytes_mm.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i32, i32, i32, vp]
        lib.qb200_qbytes_mm_quantized.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i32, i32, i32, i32, vp]
        lib.qb200_quantize_affine.argtypes = [vp, vp, vp, vp, i64, i64, i32, i32, i32, i32, vp]
        lib.qb200_pack.argtypes = [vp, vp, i64, i64, i32, vp]
        lib.qb200_quantize_qbits_max.argtypes = [vp, vp, vp, vp, i64, i64, i32, i32, i32, i32, vp]
        lib.qb200_absmax.argtypes = [vp, vp, vp, i64, i32, vp]
        lib.qb200_quantize_qbytes_absmax.argtypes = [vp, vp, vp, i64, i64, i32, i32, vp]
        lib.qb200_qbits_mm_grad_input.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i32, i32, i32, vp]
        lib.qb200_qbytes_mm_grad_input.argtypes = [vp, vp, vp, vp, i64, i64, i64, i32, i32, vp]
        f64 = ctypes.c_double
        lib.qb200_quantize_qbits_hqq.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i32, i32, i32, i32, f64, f64, f64,
                                                 i32, vp]
        lib.qb200_quantize_qbits_hqq_workspace_bytes.argtypes = [i64, i64, i32, i32]
        lib.qb200_quantize_qbits_hqq_workspace_bytes.restype = i64
        lib.qb200_hqq_shrink.argtypes = [vp, vp, i64, f64, f64, i32, vp]
        lib.qb200_qbytes_bmm.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i64, i64, i64, i64, i32, i32, vp]
        lib.qb200_qbytes_bmm_workspace_bytes.argtypes = [i64, i64, i64, i64, i32]
        lib.qb200_qbytes_bmm_workspace_bytes.restype = i64
        lib.qb200_qbytes_softmax.argtypes = [vp, vp, vp, vp, i64, i64, i32, i32, vp]
        lib.qb200_qbits_conv2d.argtypes = [vp, vp, vp, vp, vp, vp] + [i64] * 7 + [i32] * 10 + [vp]
        lib.qb200_qbytes_conv2d.argtypes = [vp, vp, vp, vp, vp] + [i64] * 7 + [i32] * 8 + [vp]
        lib.qb200_layer_norm.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, f64, i32, i32, i32, i32, vp]
        lib.qb200_absmax_update.argtypes = [vp, vp, vp, i64, i32, f64, f64, vp]
        for name in EXPORTS:
            getattr(lib, name)  # AttributeError here == header and library out of sync
        # Developer knock-outs exist only in a `make KNOCKOUTS=1` build and are set explicitly through
        # qb200_debug_set_flags by the tools that use them: no environment variable steers the library.
        _lib = lib
    return _lib


class test_override:
    """`with test_override(key, value):` -- pick one of several equivalent kernels for the calls inside (tests only)."""

    def __init__(self, key: int, value: int):
        self.key, self.value = key, value

    def __enter__(self):
        check(load().qb200_test_override(self.key, self.value), "test_override")
        return self

    def __exit__(self, *exc):
        load().qb200_test_override(self.key, 0)
        return False


def check(status: int, what: str):
    if status == 0:
        return
    msg = load().qb200_last_error().decode("utf-8", "replace")
    text = f"{what}: {ERR_NAMES.get(status, status)}: {msg}"
    if status == 2:
        raise UnsupportedConfiguration(text)
    if status == 1:
        raise ValueError(text)
    raise NativeLibraryError(text)


def stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def ptr(t):
    return None if t is None else t.data_ptr()


_workspaces = {}  # (device index, stream handle or _CAPTURE) -> zeroed uint8 buffer
_outgrown = []  # buffers replaced by larger ones: never freed, a kernel in flight or a CUDA graph may still use them
_CAPTURE = "capture"


def _zeros_outside_graph_pools(index: int, nbytes: int) -> torch.Tensor:
    """A zeroed buffer from the ordinary caching allocator, zeroed before this returns.

    It is allocated on a helper thread: CUDA-graph warm-up (cudagraph trees) routes every allocation of the calling
    thread into a graph's private pool, whose blocks a later graph may reuse.  Only ever called outside a capture.
    """
    result = []

    def run():
        try:
            with torch.cuda.device(index):
                buf = torch.zeros(nbytes, dtype=torch.uint8, device=f"cuda:{index}")
                torch.cuda.current_stream(index).synchronize()
            result.append(buf)
        except BaseException as exc:  # handed to the calling thread
            result.append(exc)

    helper = threading.Thread(target=run, name="quanto-workspace")
    helper.start()
    helper.join()
    if isinstance(result[0], BaseException):
        raise result[0]
    return result[0]


def workspace(device, stream_handle: int, nbytes: int):
    """Zero-initialised scratch for the stream-K small-M kernel; grown on demand.

    The kernel leaves the ticket counters zero on exit, so a buffer is zeroed only when allocated.  Eager calls use one
    buffer per (device, stream).  A call inside a CUDA-graph capture uses the device's capture buffer, which the eager
    calls keep as large as the largest workspace they needed; a capture never allocates one.  Every buffer comes from the
    ordinary allocator, never from a graph's pool, and is never freed, so the address a graph recorded stays valid and
    is never handed to anything else.  Graphs replayed concurrently on different streams of one device would share the
    capture buffer: replay them in order.
    """
    if nbytes <= 0:
        return None
    index = device.index if device.index is not None else torch.cuda.current_device()
    capturing = torch.cuda.is_current_stream_capturing()
    key = (index, _CAPTURE if capturing else stream_handle)
    ws = _workspaces.get(key)
    if ws is not None and ws.numel() >= nbytes:
        return ws
    if capturing:
        raise NativeLibraryError(
            f"quanto::qbits_mm: a CUDA-graph capture needs a {nbytes}-byte stream-K workspace that no call outside the "
            "capture has prepared: run the captured code once before capturing it (a warm-up)")
    for k in (key, (index, _CAPTURE)):
        old = _workspaces.get(k)
        if old is None or old.numel() < nbytes:
            if old is not None:
                _outgrown.append(old)
            _workspaces[k] = _zeros_outside_graph_pools(index, max(nbytes, 1 << 20))
    return _workspaces[key]
