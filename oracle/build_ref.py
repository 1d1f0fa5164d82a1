"""Compile the REFERENCE's own CUDA extensions for sm_90a into oracle/_ref/ (git-ignored).

TEST / BASELINE INFRASTRUCTURE.  Sources are compiled where they lie under /root/reference (never copied); the flags of the
stock setup.py files (mamba/setup.py:108-114, causal-conv1d/setup.py:107-113) are restated here with the one architecture this
project targets, -gencode arch=compute_90a,code=sm_90a.  Outputs: oracle/_ref/selective_scan_cuda.so, oracle/_ref/causal_conv1d_cuda.so
-- the GPU-side "beat this" baseline (BASELINE.md section 3a) and a second, independent GPU oracle.
Needs the reference checkout (SMB_REFERENCE_DIR, default /root/reference):  python oracle/build_ref.py
"""
import glob
import os
import shutil
import sys

REF = os.environ.get("SMB_REFERENCE_DIR", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")


def main():
    if not os.path.isdir(REF):
        print("build_ref:", REF, "not present, nothing to do")
        return 0
    os.makedirs(OUT, exist_ok=True)
    os.environ.setdefault("CC", "/usr/bin/gcc")
    os.environ["CXX"] = "/usr/bin/g++"
    os.environ.setdefault("MAX_JOBS", str(os.cpu_count() or 4))
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    from torch.utils.cpp_extension import load
    nvcc = ["-O3", "-std=c++17", "--use_fast_math", "--expt-relaxed-constexpr", "--expt-extended-lambda", "-lineinfo",
            "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__", "-U__CUDA_NO_BFLOAT16_OPERATORS__",
            "-U__CUDA_NO_BFLOAT16_CONVERSIONS__", "-U__CUDA_NO_BFLOAT162_OPERATORS__", "-U__CUDA_NO_BFLOAT162_CONVERSIONS__",
            "-gencode", "arch=compute_90a,code=sm_90a", "-ccbin", "/usr/bin/g++"]
    jobs = [
        ("selective_scan_cuda", os.path.join(REF, "mamba", "csrc", "selective_scan"),
         ["selective_scan.cpp"] + sorted(os.path.basename(p) for p in glob.glob(os.path.join(REF, "mamba", "csrc", "selective_scan", "*.cu")))),
        ("causal_conv1d_cuda", os.path.join(REF, "causal-conv1d", "csrc"),
         ["causal_conv1d.cpp", "causal_conv1d_fwd.cu", "causal_conv1d_bwd.cu", "causal_conv1d_update.cu"]),
    ]
    for name, d, files in jobs:
        target = os.path.join(OUT, name + ".so")
        if os.path.exists(target):
            print("build_ref:", target, "exists")
            continue
        bdir = os.path.join(OUT, "_build", name)           # scratch inside the git-ignored output directory, removed below
        os.makedirs(bdir, exist_ok=True)
        load(name=name, sources=[os.path.join(d, f) for f in files], extra_include_paths=[d], extra_cflags=["-O3", "-std=c++17"],
             extra_cuda_cflags=nvcc, build_directory=bdir, verbose=False, is_python_module=False)
        shutil.copy(os.path.join(bdir, name + ".so"), target)
        shutil.rmtree(os.path.join(OUT, "_build"), ignore_errors=True)
        print("build_ref: built", target)
    return 0


if __name__ == "__main__":
    sys.exit(main())
