"""Build the C-ABI shared library libdojo_b200.so in-tree with nvcc for sm_90a (H100).

    python -m dojo_jl_b200.build        (or __graft_entry__.build())
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdojo_b200.so")
SOURCES = ["dojo_b200.cu", "dojo_b200_cm.cu"]
HEADERS = ["dojo_step_kernel.cuh", "dojo_contact_orthant.cuh", "dojo_joint_tra.cuh", "dojo_kernels.cuh", "dojo_grad.cuh", "dojo_kin.cuh", "dojo_kinjac.cuh", "dojo_envs.cuh", "dojo_storage.cuh", "dojo_lqr.cuh", "dojo_linalg.cuh", "dojo_math.cuh", "dojo_plan.h", os.path.join("..", "..", "include", "dojo_b200.h")]


def nvcc_path() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the CUDA toolkit is required to build libdojo_b200.so")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    # this file counts as a source: a library compiled with other flags (another architecture) is rebuilt
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, defines=(), out: str = LIB) -> str:
    if not force and not needs_build() and out == LIB:
        return LIB
    cmd = [nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-maxrregcount=255",
           "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-shared", "-o", out + ".tmp"] + \
          [f"-D{d}" for d in defines] + [os.path.join(CSRC, s) for s in SOURCES]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.check_call(cmd)
    os.replace(out + ".tmp", out)  # never leave a half-written library in the tree
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
