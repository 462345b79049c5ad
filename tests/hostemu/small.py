"""The forward kernel specialised for small mechanisms on the CPU -- TEST INFRASTRUCTURE for tests/test_small_step.py.

SmallEmu builds the kernel emulation TU of gen.py (generated from the unmodified sources, like tests/hostemu/trace.py) with two more
entry points: hostemu_step_small runs dojo_step_kernel<false, true, false, SMALL = true> on CPU fibers, and hostemu_small_step_ok
evaluates the product's selection rule (dojo_b200.cu, small_step_ok) for the handle.  The library is built into tests/hostemu/_build
(or a temporary directory when the tree is read-only)."""
import ctypes as C
import os

import numpy as np

from dojo_jl_b200 import capi
from . import gen
from .harness import HostEmu, _ip, _p, _vp
from .trace import _build_dir, _compile, _stale, _substitute

_EMU_ENTRY = r"""
// dojo_step / dojo_rollout on the emulation with the forward kernel dojo_create picks for small mechanisms (plan in shared memory)
extern "C" int hostemu_step_small(void* p, const DojoSolverOptions* opts, int B, int T, const double* Z, const double* U, const double* Fext, double* Zn,
                                  double* sol, int32_t* status, int32_t* iters, uint32_t flags, int slots, int grid, double* traj) {
  DojoHandle* h = static_cast<EmuHandle*>(p)->h;
  int counter = 0;
  StepArgs a = emu_args(h, opts, B, false, slots, true, &counter);
  a.Z = Z; a.U = U; a.Fext = Fext; a.Zn = Zn; a.sol = sol; a.status = status; a.iters = iters; a.flags = flags; a.T = T; a.traj = traj;
  const size_t smem = slots * h->arena_bytes + h->blob_bytes;
  for (int b = 0; b < grid; ++b) emu::run_cta(b, grid, 32 * h->nw * slots, smem, [&a] { dojo_step_kernel<false, true, false, true>(a); });
  return 0;
}
// small_step_ok of dojo_create, with the plan placement dojo_create computes from the device (smem_plan: every table in shared memory)
extern "C" int hostemu_small_step_ok(void* p, int smem_plan) { return small_step_ok(static_cast<EmuHandle*>(p)->h, smem_plan ? 0xff : 0) ? 1 : 0; }
"""


def build_emulation() -> str:
    name = "libdojo_hostemu_small_fma.so" if gen.FMA else "libdojo_hostemu_small.so"
    lib = os.path.join(_build_dir(), name)
    if not _stale(lib, gen.DEPS + [os.path.abspath(__file__)]):
        return lib
    here = gen.HERE
    text = open(gen.generate()).read()
    text = _substitute(text, [('#include "../cuda_shim.h"', f'#include "{os.path.join(here, "cuda_shim.h")}"'),
                              ('#include "../driver.inc"', f'#include "{os.path.join(here, "driver.inc")}"')], "the emulation TU")
    fp = ["-ffp-contract=fast", "-march=x86-64-v3"] if gen.FMA else ["-ffp-contract=off"]
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared"] + fp + ["-Wno-unknown-pragmas", "-Wno-unused-function", "-Wno-unused-variable",
                                                                         "-Wno-unused-but-set-variable"]
    return _compile(text + _EMU_ENTRY, name, cmd)


class SmallEmu(HostEmu):
    """HostEmu's generic kernels (step, step_grad) and the forward kernel specialised for small mechanisms (step_small) in one library."""

    def __init__(self, mech):
        L = C.CDLL(build_emulation())
        op = C.POINTER(capi.DojoSolverOptions)
        L.hostemu_step_small.argtypes = [_vp, op, _ip, _ip, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint32, _ip, _ip, _vp]
        L.hostemu_step_small.restype = C.c_int
        L.hostemu_small_step_ok.argtypes = [_vp, _ip]
        L.hostemu_small_step_ok.restype = C.c_int
        L.hostemu_create.restype = _vp
        L.hostemu_create.argtypes = [C.POINTER(capi.DojoMechanismDesc)]
        L.hostemu_destroy.argtypes = [_vp]
        L.hostemu_last_error.restype = C.c_char_p
        for n in ("hostemu_num_residual", "hostemu_num_input", "hostemu_warps_per_env"):
            getattr(L, n).argtypes = [_vp]
        L.hostemu_step.argtypes = [_vp, op, _ip, _ip, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint32, _ip, _ip, _ip, _vp]
        self.L, self.mech = L, mech
        desc, self._keep = capi.flatten(mech)
        h = L.hostemu_create(C.byref(desc))
        if not h:
            raise RuntimeError("hostemu_create failed: " + L.hostemu_last_error().decode())
        self.h = C.c_void_p(h)
        assert L.hostemu_num_residual(self.h) == mech.nres

    def small_step_ok(self, smem_plan=True) -> bool:
        """dojo_create's choice of the specialised forward kernel for this mechanism (reads the DOJO_B200_* switches like dojo_create)"""
        return bool(self.L.hostemu_small_step_ok(self.h, int(smem_plan)))

    def step_small(self, Z, U=None, opts=None, T=1, fext=None, flags=0, slots=1, grid=1, record=False):
        """HostEmu.step with the specialised kernel.  Returns (Z_next, status, iters, sol[, traj])."""
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=np.float64)
        B = Z.shape[0]
        if U is not None:
            U = np.ascontiguousarray(U, dtype=np.float64)
        Zn = np.empty_like(Z)
        sol = np.empty((B, self.mech.nres))
        st, it = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        traj = np.empty((T, B, Z.shape[1])) if record else None
        o = opts if opts is not None else capi.solver_options()
        self.L.hostemu_step_small(self.h, C.byref(o), B, T, _p(Z), _p(U), _p(fext), _p(Zn), _p(sol), _p(st), _p(it), flags, slots, grid, _p(traj))
        return (Zn, st, it, sol, traj) if record else (Zn, st, it, sol)
