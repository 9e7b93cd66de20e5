"""Run the reference's OWN hot-path tests against the sm_90a kernels (SURVEY 4: "still pass the reference's tests").

Needs oracle/_ref (python oracle/build_ref.py in the authoring container: the unmodified reference + its tests, git-ignored,
travels to the GPU box).  The kernels are bound into the real `optimum.quanto` classes by quanto_b200.integration.

    python tools/run_reference_tests.py [--cpu] [extra pytest args]

Selected tests (reference paths): tests/library/test_unpack.py, test_quantize.py, test_mm.py::test_qbytes_mm,
tests/tensor/test_packed_tensor.py, tests/tensor/ops/test_linear_dispatch.py, tests/tensor/weights (canonical classes),
tests/tensor/optimizers/test_hqq_optimizer.py, tests/nn/test_qlinear.py, and the quantized-attention tests
tests/tensor/ops/test_mm_dispatch.py, tests/tensor/activations/test_activations_dispatch.py, tests/nn/test_qattention.py,
the quantized convolution tests tests/nn/test_qconv2d.py and the quantized layer norm tests tests/nn/test_qlayernorm.py.
The tests of the retired AWQ / Marlin / TinyGemm
bindings are deselected (those ops are no longer reached; INTEGRATION.md)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
TESTS = os.path.join(REF, "reference_tests")


def main():
    if not os.path.isdir(TESTS):
        raise SystemExit("oracle/_ref is missing: run `python oracle/build_ref.py` where /root/reference exists")
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([REF, os.path.join(ROOT, "optimum-quanto_b200"), os.path.join(ROOT, "tools"),
                                         env.get("PYTHONPATH", "")])
    env["TORCH_CUDA_ARCH_LIST"] = "9.0"
    sel = ["library/test_unpack.py", "library/test_quantize.py", "library/test_mm.py::test_qbytes_mm",
           "tensor/test_packed_tensor.py", "tensor/ops/test_linear_dispatch.py",
           "tensor/weights/test_weight_qbits_tensor_dispatch.py", "tensor/weights/test_weight_qbits_tensor_quantize.py",
           "tensor/weights/test_weight_qbytes_tensor_dispatch.py", "tensor/weights/test_weight_qbytes_tensor_quantize.py",
           "tensor/optimizers/test_hqq_optimizer.py", "nn/test_qlinear.py",
           "tensor/ops/test_mm_dispatch.py", "tensor/activations/test_activations_dispatch.py", "nn/test_qattention.py",
           "nn/test_qconv2d.py", "nn/test_qlayernorm.py"]
    extra = [a for a in sys.argv[1:] if a != "--cpu"]
    cmd = [sys.executable, "-m", "pytest", "-q", "-p", "quanto_b200_bind", "-x" if "--cpu" in sys.argv else "--maxfail=50",
           "--deselect", "nn/test_qlinear.py::test_qlinear_gradient"] + sel + extra
    return subprocess.run(cmd, cwd=TESTS, env=env).returncode


if __name__ == "__main__":
    sys.exit(main())
