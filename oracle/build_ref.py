"""Recipe for oracle/_ref: the UNMODIFIED reference installed from /root/reference (authoring container only).

TEST / BENCH INFRASTRUCTURE, git-ignored, never imported by the product.  `pip install --target oracle/_ref` of the
reference (its wheel omits the JIT extension sources, which are overlaid from the same tree), its own tests and bench
scripts beside it, and its two JIT extensions pre-built here so that the GPU box (same image, no /root/reference, no
network) can import them without compiling: `quanto_cpp` (CPU unpack) and `quanto_cuda` (unpack, AWQ v2, Marlin int4 /
fp8 -- the kernels the reference itself would dispatch to on an H100, SURVEY 2.2), cross-compiled for sm_90.

Used by: bench.py --impl reference (kind "reference" when importable), tools/run_reference_tests.py (the reference's
own hot-path tests against the sm_90a ops).

    python oracle/build_ref.py [--cuda]
"""
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
SRC = "/root/reference"


def main():
    if not os.path.isdir(SRC):
        raise SystemExit("the reference tree is only present in the authoring container")
    if not os.path.isdir(os.path.join(REF, "optimum")):
        tmp = "/tmp/refcopy"
        shutil.rmtree(tmp, ignore_errors=True)
        shutil.copytree(SRC, tmp)
        subprocess.run([sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps",
                        "--find-links", "/opt/wheelhouse", "--target", REF, tmp], check=True)
        ext = "optimum/quanto/library/extensions"
        shutil.copytree(os.path.join(SRC, ext), os.path.join(REF, ext), dirs_exist_ok=True)
        shutil.copytree(os.path.join(SRC, "tests"), os.path.join(REF, "reference_tests"), dirs_exist_ok=True)
        shutil.copytree(os.path.join(SRC, "bench"), os.path.join(REF, "reference_bench"), dirs_exist_ok=True)
    sys.path.insert(0, REF)
    import torch
    import optimum.quanto  # noqa: F401
    # CPU extension: first use builds it into <ext dir>/build
    packed = torch.randint(0, 255, (4, 8), dtype=torch.uint8)
    torch.ops.quanto.unpack(packed, 4)
    print("quanto_cpp built")
    if "--cuda" in sys.argv:
        os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0"
        from torch.utils.cpp_extension import load
        root = os.path.join(REF, "optimum/quanto/library/extensions/cuda")
        sources = ["unpack.cu", "awq/v2/gemm_cuda.cu", "awq/v2/gemv_cuda.cu", "marlin/fp8_marlin.cu",
                   "marlin/gptq_marlin_repack.cu", "marlin/marlin_cuda.cpp", "marlin/marlin_cuda_kernel.cu",
                   "pybind_module.cpp"]
        build = os.path.join(root, "build")
        os.makedirs(build, exist_ok=True)
        # the flags of optimum/quanto/library/extensions/cuda/__init__.py:47-55 on an H100 (capability 9.0 -> "900")
        load(name="quanto_cuda", sources=[f"{root}/{s}" for s in sources], extra_cflags=["-g", "-O3"],
             extra_cuda_cflags=["--expt-extended-lambda", "--use_fast_math", "-DQUANTO_CUDA_ARCH=900"],
             build_directory=build, verbose=True)
        with open(os.path.join(build, "pytorch_version.txt"), "w") as f:
            f.write(torch.__version__)
        print("quanto_cuda built for sm_90")


if __name__ == "__main__":
    main()
