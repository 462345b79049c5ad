"""The forward kernel specialised for small mechanisms on the CPU -- TEST INFRASTRUCTURE for tests/test_small_step.py.

SmallEmu reaches two more entry points of the kernel emulation (driver.inc): hostemu_step_small runs dojo_step_kernel<false, true,
false, SMALL = true> on CPU fibers, and hostemu_small_step_ok evaluates the product's selection rule (dojo_b200.cu,
small_step_ok) for the handle."""
import ctypes as C

import numpy as np

from dojo_jl_b200 import capi
from .harness import HostEmu, _p


class SmallEmu(HostEmu):
    """HostEmu's generic kernels (step, step_grad) and the forward kernel specialised for small mechanisms (step_small)."""

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
