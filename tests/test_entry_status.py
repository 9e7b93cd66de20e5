"""The status contract of the C-ABI entry points of the elementwise, freeze, HQQ, layer-norm and softmax kernels.

Every call runs in a subprocess whose CUDA runtime sees no device (CUDA_VISIBLE_DEVICES empty), so the dummy device
pointers below are never launched on or dereferenced:
  - a bad argument returns its documented code (QB200_ERR_ARG / QB200_ERR_UNSUPPORTED) before any CUDA call;
  - a valid call reaches the runtime, which fails: QB200_ERR_CUDA, and qb200_last_error names the op and carries the
    runtime's reason.
"""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARG, UNSUP, CUDA = 1, 2, 3
F32, F16, BF16, I8, U8, E4M3, E5M2, E4M3FNUZ = range(8)
P = 1 << 20      # dummy device address, 256-byte aligned
NULL = None
# cudaGetErrorString of cudaErrorNoDevice (no visible GPU) / cudaErrorInsufficientDriver (no driver installed)
RUNTIME_REASONS = ("no CUDA-capable device", "CUDA driver version is insufficient")

# (entry point, arguments without the trailing stream): valid calls
VALID = {
    "unpack": ("qb200_unpack", [P, P, 64, 4]),
    "pack": ("qb200_pack", [P, P, 8, 16, 4]),
    "quantize_symmetric": ("qb200_quantize_symmetric", [P, P, P, 4, 64, 0, BF16, I8]),
    "quantize_affine": ("qb200_quantize_affine", [P, P, P, P, 4, 64, 1, 4, BF16, 0]),
    "dequantize_qbits": ("qb200_dequantize_qbits", [P, P, P, P, 8, 128, 64, 4, BF16, 0]),
    "quantize_qbits_max": ("qb200_quantize_qbits_max", [P, P, P, P, 8, 128, 64, 4, BF16, 0]),
    "absmax": ("qb200_absmax", [P, P, P, 64, BF16]),
    "absmax_update": ("qb200_absmax_update", [P, P, P, 64, BF16, 127.0, 0.9]),
    "quantize_qbytes_absmax": ("qb200_quantize_qbytes_absmax", [P, P, P, 8, 64, BF16, I8]),
    "quantize_qbits_hqq": ("qb200_quantize_qbits_hqq", [P, P, P, P, P, P, 8, 128, 64, 4, BF16, 0, 0.7, 10.0, 1.01, 3]),
    "hqq_shrink": ("qb200_hqq_shrink", [P, P, 64, 10.0, 0.7, BF16]),
    "layer_norm": ("qb200_layer_norm", [P, NULL, NULL, NULL, P, P, 4, 64, 1e-5, BF16, BF16, I8, F32]),
    "qbytes_softmax": ("qb200_qbytes_softmax", [P, P, P, P, 4, 64, I8, BF16]),
}


def _with(op, **changes):
    """The valid call of `op` with arguments replaced by position: _with("unpack", a3=3) sets argument 3 to 3."""
    fn, args = VALID[op]
    args = list(args)
    for key, value in changes.items():
        args[int(key[1:])] = value
    return fn, args


# (case id, expected status, call)
REJECTED = [
    ("unpack-bits", ARG, _with("unpack", a3=3)),
    ("unpack-negative-size", ARG, _with("unpack", a2=-1)),
    ("unpack-null", ARG, _with("unpack", a1=NULL)),
    ("pack-bits", ARG, _with("pack", a4=8)),
    ("pack-negative-shape", ARG, _with("pack", a2=-1)),
    ("pack-null", ARG, _with("pack", a0=NULL)),
    ("quantize_symmetric-input-dtype", ARG, _with("quantize_symmetric", a6=I8)),
    ("quantize_symmetric-target-dtype", ARG, _with("quantize_symmetric", a7=F16)),
    ("quantize_symmetric-axis", ARG, _with("quantize_symmetric", a5=3)),
    ("quantize_symmetric-negative-shape", ARG, _with("quantize_symmetric", a3=-1)),
    ("quantize_affine-bits", ARG, _with("quantize_affine", a7=0)),
    ("quantize_affine-axis", ARG, _with("quantize_affine", a6=3)),
    ("quantize_affine-null", ARG, _with("quantize_affine", a2=NULL)),
    ("quantize_affine-dtype", ARG, _with("quantize_affine", a8=I8)),
    ("dequantize_qbits-bits", ARG, _with("dequantize_qbits", a7=3)),
    ("dequantize_qbits-group", ARG, _with("dequantize_qbits", a6=6)),
    ("dequantize_qbits-shape", ARG, _with("dequantize_qbits", a4=0)),
    ("dequantize_qbits-packed-alignment", ARG, _with("dequantize_qbits", a0=P + 2)),
    ("dequantize_qbits-out-alignment", ARG, _with("dequantize_qbits", a3=P + 8)),
    ("dequantize_qbits-dtype", ARG, _with("dequantize_qbits", a8=I8)),
    ("quantize_qbits_max-bits", ARG, _with("quantize_qbits_max", a7=8)),
    ("quantize_qbits_max-group-divides-k", ARG, _with("quantize_qbits_max", a6=48)),
    ("quantize_qbits_max-group", UNSUP, _with("quantize_qbits_max", a5=120, a6=12)),
    ("quantize_qbits_max-null", ARG, _with("quantize_qbits_max", a3=NULL)),
    ("quantize_qbits_max-alignment", UNSUP, _with("quantize_qbits_max", a0=P + 8)),
    ("quantize_qbits_max-dtype", ARG, _with("quantize_qbits_max", a8=I8)),
    ("absmax-negative-size", ARG, _with("absmax", a3=-1)),
    ("absmax-null", ARG, _with("absmax", a2=NULL)),
    ("absmax-scratch-alignment", ARG, _with("absmax", a2=P + 2)),
    ("absmax_update-empty", ARG, _with("absmax_update", a3=0)),
    ("absmax_update-null", ARG, _with("absmax_update", a1=NULL)),
    ("absmax_update-scratch-alignment", ARG, _with("absmax_update", a2=P + 2)),
    ("absmax_update-qmax", ARG, _with("absmax_update", a5=0.0)),
    ("absmax_update-dtype", ARG, _with("absmax_update", a4=I8)),
    ("quantize_qbytes_absmax-negative-shape", ARG, _with("quantize_qbytes_absmax", a3=-1)),
    ("quantize_qbytes_absmax-null", ARG, _with("quantize_qbytes_absmax", a2=NULL)),
    ("quantize_qbytes_absmax-target-dtype", ARG, _with("quantize_qbytes_absmax", a6=E4M3FNUZ)),
    ("quantize_qbytes_absmax-dtype", ARG, _with("quantize_qbytes_absmax", a5=I8)),
    ("quantize_qbits_hqq-bits", ARG, _with("quantize_qbits_hqq", a9=3)),
    ("quantize_qbits_hqq-shape", ARG, _with("quantize_qbits_hqq", a7=0)),
    ("quantize_qbits_hqq-iters", ARG, _with("quantize_qbits_hqq", a15=-1)),
    ("quantize_qbits_hqq-f32", UNSUP, _with("quantize_qbits_hqq", a10=F32)),
    ("quantize_qbits_hqq-dtype", ARG, _with("quantize_qbits_hqq", a10=I8)),
    ("quantize_qbits_hqq-cube", UNSUP, _with("quantize_qbits_hqq", a12=4.0)),
    ("quantize_qbits_hqq-group", UNSUP, _with("quantize_qbits_hqq", a7=120, a8=12)),
    ("quantize_qbits_hqq-too-many-iters", UNSUP, _with("quantize_qbits_hqq", a15=65)),
    ("quantize_qbits_hqq-null", ARG, _with("quantize_qbits_hqq", a5=NULL)),
    ("quantize_qbits_hqq-workspace-alignment", UNSUP, _with("quantize_qbits_hqq", a5=P + 16)),
    ("hqq_shrink-negative-size", ARG, _with("hqq_shrink", a2=-1)),
    ("hqq_shrink-f32", UNSUP, _with("hqq_shrink", a5=F32)),
    ("hqq_shrink-dtype", ARG, _with("hqq_shrink", a5=I8)),
    ("hqq_shrink-null", ARG, _with("hqq_shrink", a1=NULL)),
    ("layer_norm-shape", ARG, _with("layer_norm", a7=0)),
    ("layer_norm-dtype", ARG, _with("layer_norm", a10=I8)),
    ("layer_norm-input-dtype", ARG, _with("layer_norm", a9=U8)),
    ("layer_norm-output-dtype", ARG, _with("layer_norm", a11=F16)),
    ("layer_norm-codes-in-without-scale", ARG, _with("layer_norm", a9=I8)),
    ("layer_norm-codes-out-without-scale", ARG, _with("layer_norm", a4=NULL)),
    ("layer_norm-output-scale-dtype", ARG, _with("layer_norm", a12=I8)),
    ("layer_norm-eps", ARG, _with("layer_norm", a8=-1.0)),
    ("qbytes_softmax-shape", ARG, _with("qbytes_softmax", a5=0)),
    ("qbytes_softmax-code-dtype", ARG, _with("qbytes_softmax", a6=F16)),
    ("qbytes_softmax-null", ARG, _with("qbytes_softmax", a1=NULL)),
]

_SCRIPT = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from quanto_b200 import _native
lib = _native.load()
out = []
for fn, args in json.loads(sys.stdin.read()):
    rc = getattr(lib, fn)(*args, None)
    out.append([rc, lib.qb200_last_error().decode()])
print(json.dumps(out))
"""


@pytest.fixture(scope="module")
def no_device_results():
    """{case id: (status, qb200_last_error)} of every call, made in one process that sees no CUDA device."""
    cases = [(op, VALID[op]) for op in VALID] + [(cid, call) for cid, _, call in REJECTED]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    proc = subprocess.run([sys.executable, "-c", _SCRIPT, os.path.join(ROOT, "optimum-quanto_b200")],
                          input=json.dumps([call for _, call in cases]), env=env, capture_output=True, text=True,
                          timeout=600)
    assert proc.returncode == 0, proc.stderr
    results = json.loads(proc.stdout.strip().splitlines()[-1])
    return {cid: tuple(r) for (cid, _), r in zip(cases, results)}


@pytest.mark.parametrize("cid,expected", [(cid, expected) for cid, expected, _ in REJECTED])
def test_bad_arguments_return_the_documented_status(no_device_results, cid, expected):
    rc, msg = no_device_results[cid]
    assert rc == expected, (rc, msg)
    assert msg.startswith(cid.split("-")[0] + ":"), msg


@pytest.mark.parametrize("op", list(VALID))
def test_cuda_failure_names_the_op_and_the_runtime_reason(no_device_results, op):
    rc, msg = no_device_results[op]
    assert rc == CUDA, (rc, msg)
    assert msg.startswith(op + ":") or msg.startswith(op + " "), msg
    assert any(reason in msg for reason in RUNTIME_REASONS), msg

