"""The traced step on the CPU -- TEST INFRASTRUCTURE for tests/test_solver_trace.py and tests/test_zzzzz_gpu_solver_trace.py.

  * TracedEmu: the kernel emulation (gen.py) through its entry point hostemu_step_trace (driver.inc), which runs the product's traced
    kernel dojo_step_kernel<false, false, true> on CPU fibers.
  * TracedOracle: the CPU oracle (oracle/dojo_oracle.cpp) with its loop-head record extended by a fifth column, the trials the previous
    iteration's line_search evaluated up to and including the accepted one, so that its rows can be compared with the device's
    [rvio, bvio, alpha, mu, trials] (include/dojo_b200.h, dojo_step_trace).  Five textual substitutions, each asserted to apply exactly
    once; they add integer bookkeeping only, and the tests check that its steps stay bit-identical to the oracle's.  Built from the
    unmodified source into the emulation's build directory (gen.build_dir)."""
import ctypes as C
import os
import subprocess

import numpy as np

from dojo_jl_b200 import capi
from oracle import oracle as _oracle
from . import gen
from .harness import HostEmu, _p

ROOT = gen.ROOT
ORACLE_DIR = os.path.join(ROOT, "oracle")


_build_dir, _stale = gen.build_dir, gen.stale


def _compile(src_text, name, cmd):
    d = _build_dir()
    lib = os.path.join(d, name)
    src = lib[:-3] + ".cpp"
    with open(src, "w") as f:
        f.write(src_text)
    subprocess.check_call(cmd + ["-o", lib + ".tmp", src])
    os.replace(lib + ".tmp", lib)
    return lib


def _substitute(text, subs, what):
    for a, b in subs:
        if text.count(a) != 1:
            raise RuntimeError(f"expected exactly one occurrence of {a!r} in {what}")
        text = text.replace(a, b)
    return text


# ---------------------------------------------------------------------------------------------------------------- kernel emulation
class TracedEmu(HostEmu):
    """HostEmu's untraced step (step) and the traced one (step_trace)."""

    def step_trace(self, Z, U=None, opts=None, fext=None, flags=0, slots=1, smem_plan=True, grid=1):
        """dojo_step_trace.  Returns (Z_next, status, iters, sol, trace [B, max_iter, 5])."""
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=np.float64)
        B = Z.shape[0]
        if U is not None:
            U = np.ascontiguousarray(U, dtype=np.float64)
        o = opts if opts is not None else capi.solver_options()
        Zn = np.empty_like(Z)
        sol = np.empty((B, self.mech.nres))
        st, it = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        trace = np.empty((B, max(o.max_iter, 0), 5))
        self.L.hostemu_step_trace(self.h, C.byref(o), B, _p(Z), _p(U), _p(fext), _p(Zn), _p(sol), _p(st), _p(it), _p(trace), flags, slots,
                                  int(smem_plan), grid)
        return Zn, st, it, sol, trace


# ---------------------------------------------------------------------------------------------------------------- oracle
_ORACLE_SUBS = [
    # the trial counter: reset with the record of every solve, set by every candidate line_search evaluates
    ("  int force_iters = -1;\n", "  int force_iters = -1;\n  int ls_trials = 0;  // trials of the last line_search up to the accepted one\n"),
    ("    trace.clear();\n", "    trace.clear();\n    ls_trials = 0;\n"),
    ("      candidate_step(alpha, scale);\n", "      candidate_step(alpha, scale);\n      ls_trials = n + 1;\n"),
    # the fifth column of every loop-head row, and the row count of oracle_trace
    ("trace.push_back(mutarget);", "trace.push_back(mutarget); trace.push_back(ls_trials);"),
    ("return (int)o->trace.size() / 4;", "return (int)o->trace.size() / 5;"),
]


def build_oracle() -> str:
    name = "libdojo_oracle_trace.so"
    src = os.path.join(ORACLE_DIR, "dojo_oracle.cpp")
    deps = [src, os.path.join(ORACLE_DIR, "dojo_math.hpp"), os.path.join(ROOT, "include", "dojo_b200.h"), os.path.abspath(__file__)]
    lib = os.path.join(_build_dir(), name)
    if not _stale(lib, deps):
        return lib
    text = _substitute(open(src).read(), _ORACLE_SUBS, "oracle/dojo_oracle.cpp")
    # the flags of oracle/Makefile; the oracle's own directory first on the include path, so that its relative includes resolve
    cmd = ["g++", "-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-pthread", "-shared", "-I", ORACLE_DIR]
    return _compile(text, name, cmd)


_oracle_lib = None


def _traced_oracle_lib():
    global _oracle_lib
    if _oracle_lib is None:
        base = _oracle.lib()  # argument types of every entry point, as oracle.py declares them
        L = C.CDLL(build_oracle())
        for n in dir(base):
            if n.startswith("oracle_"):
                f, g = getattr(base, n), getattr(L, n)
                g.argtypes, g.restype = f.argtypes, f.restype
        _oracle_lib = L
    return _oracle_lib


class TracedOracle(_oracle.Oracle):
    """Oracle whose trace() has five columns: (rvio, bvio, alpha, mu, trials) per loop head, alpha / mu / trials of the previous iteration."""

    def __init__(self, mech, opts=None):
        self.mech = mech
        self.L = _traced_oracle_lib()
        desc, self._keep = capi.flatten(mech)
        self.h = C.c_void_p(self.L.oracle_create(C.byref(desc)))
        self.nres = self.L.oracle_num_residual(self.h)
        self.nu = self.L.oracle_num_input(self.h)
        assert self.nres == mech.nres and self.nu == mech.nu
        self.opts = opts if opts is not None else capi.solver_options()

    def trace(self):
        n = self.L.oracle_trace(self.h, None, 0)
        buf = np.empty(5 * n)
        self.L.oracle_trace(self.h, _oracle._d(buf), buf.size)
        return buf.reshape(n, 5)
