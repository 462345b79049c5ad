"""Reverse mode through a fused rollout on the CPU -- TEST INFRASTRUCTURE for tests/test_rollout_vjp.py.

VjpEmu runs, on CPU fibers, the two launches of dojo_rollout_tape / dojo_rollout_vjp: the recording rollout
dojo_step_kernel<false, ..., REC = true> without the gradient kernel (the tape is its sol_raw), and the adjoint kernel
dojo_step_kernel<true, ..., VJP = true>.  Its entry points are appended to the emulation's generated translation unit (gen.generate(): the
product's kernel, handle and table builder with driver.inc), which is compiled into a library of its own, as feedback.py does; so VjpEmu
also has every entry point of HostEmu and rollout_grad.py's rollout_grad, and the Jacobians it is compared with come from the same library.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from dojo_jl_b200 import capi
from . import gen
from .feedback import _patched
from .harness import _ip, _p, _vp
from .rollout_grad import RolloutGradEmu

ENTRY = r"""
// dojo_rollout_tape: the recording rollout (REC) without publication or gradient kernel.  traj [nz x B x (T + 1)] holds Z0 in slab 0
extern "C" int hostemu_rollout_tape(void* p, const DojoSolverOptions* opts, int B, int T, double* traj, const double* U, double* tape, int32_t* status,
                                    int32_t* iters, int slots, int smem_plan, int grid) {
  DojoHandle* h = static_cast<EmuHandle*>(p)->h;
  int counter = 0;
  StepArgs a = emu_args(h, opts, B, false, slots, smem_plan != 0, &counter);
  a.Z = traj; a.U = U; a.traj = traj + (size_t)B * h->plan.nz; a.T = T; a.sol_raw = tape; a.status = status; a.iters = iters;
  emu_launch<false, false, false, false, true>(h, a, grid, slots, smem_plan != 0);
  return 0;
}
// dojo_rollout_vjp: the adjoint kernel (VJP) in the gradient launch configuration; gZ0 carries lambda
extern "C" int hostemu_rollout_vjp(void* p, int B, int T, const double* traj, const double* U, const double* tape, const double* gZ, double* gZ0,
                                   double* gU, int32_t* status, int slots_grad, int smem_plan, int grid) {
  DojoHandle* h = static_cast<EmuHandle*>(p)->h;
  if (!h->grad_bytes) return -1;
  int counter = 0;
  StepArgs g = emu_args(h, nullptr, B, true, slots_grad, smem_plan != 0, &counter);
  g.Z = traj; g.U = U; g.sol_raw = const_cast<double*>(tape); g.status = status; g.T = T;
  g.vjp_gZ = gZ; g.vjp_lam = gZ0; g.vjp_gU = gU;
  if (smem_plan) emu_launch<true, true, false, false, false, false, true>(h, g, grid, slots_grad, true);
  else emu_launch<true, false, false, false, false, false, true>(h, g, grid, slots_grad, false);
  return 0;
}
"""


def build() -> str:
    """the emulation library with the two entry points, in a directory of its own next to gen.build()'s (same compiler flags)"""
    d = os.path.join(gen.build_dir(), "vjp")
    os.makedirs(d, exist_ok=True)
    lib = os.path.join(d, "libdojo_hostemu_vjp_fma.so" if gen.FMA else "libdojo_hostemu_vjp.so")
    if not gen.stale(lib, gen.DEPS + [os.path.abspath(__file__)]):
        return lib
    with _patched(gen, "build_dir", lambda: d):  # generate() writes its TU into d, not over the one gen.build() compiles
        tu = gen.generate()
    with open(tu, "a") as f:
        f.write(ENTRY)
    fp = ["-ffp-contract=fast", "-march=x86-64-v3"] if gen.FMA else ["-ffp-contract=off"]
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared"] + fp + ["-Wno-unknown-pragmas", "-Wno-unused-function",
                           "-Wno-unused-variable", "-Wno-unused-but-set-variable", "-o", lib + ".tmp", tu])
    os.replace(lib + ".tmp", lib)
    return lib


class VjpEmu(RolloutGradEmu):
    """HostEmu's kernels, rollout_grad, and the tape / adjoint pair (rollout_tape, rollout_vjp), all from the library of build()."""

    def __init__(self, mech):
        lib = build()
        with _patched(gen, "build", lambda: lib):  # HostEmu loads gen.build()'s library; this one is a superset of it
            super().__init__(mech)
        op = C.POINTER(capi.DojoSolverOptions)
        self.L.hostemu_rollout_tape.argtypes = [_vp, op, _ip, _ip, _vp, _vp, _vp, _vp, _vp, _ip, _ip, _ip]
        self.L.hostemu_rollout_vjp.argtypes = [_vp, _ip, _ip, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ip, _ip, _ip]

    def rollout_tape(self, Z0, U=None, T=1, opts=None, slots=1, smem_plan=True, grid=1):
        """dojo_rollout_tape, U [T, B, nu].  Returns (Z_traj [T+1, B, nz], tape [T, B, nres], status [T, B], iters [T, B])."""
        Z0 = np.ascontiguousarray(np.atleast_2d(Z0), dtype=np.float64)
        B = Z0.shape[0]
        U = None if U is None else np.ascontiguousarray(U, dtype=np.float64)
        assert U is None or U.shape == (T, B, self.mech.nu)
        traj = np.empty((T + 1, B, Z0.shape[1]))
        traj[0] = Z0
        tape = np.empty((T, B, self.mech.nres))
        st, it = np.zeros((T, B), dtype=np.int32), np.zeros((T, B), dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        self.L.hostemu_rollout_tape(self.h, C.byref(o), B, T, _p(traj), _p(U), _p(tape), _p(st), _p(it), slots, int(smem_plan), grid)
        return traj, tape, st, it

    def rollout_vjp(self, Z_traj, U, tape, gZ, slots_grad=1, smem_plan=True, grid=1, with_gU=True):
        """dojo_rollout_vjp, gZ [T+1, B, 12Nb].  Returns (gZ0 [B, 12Nb], gU [T, B, nu] or None, status [B])."""
        T, B = tape.shape[0], tape.shape[1]
        traj = np.ascontiguousarray(Z_traj, dtype=np.float64)
        U = None if U is None else np.ascontiguousarray(U, dtype=np.float64)
        gZ = np.ascontiguousarray(gZ, dtype=np.float64)
        assert gZ.shape == (T + 1, B, 12 * self.mech.Nb)
        gZ0 = np.full((B, 12 * self.mech.Nb), -1.0)
        gU = np.full((T, B, self.mech.nu), -1.0) if with_gU else None
        st = np.full(B, -1, dtype=np.int32)
        rc = self.L.hostemu_rollout_vjp(self.h, B, T, _p(traj), _p(U), _p(np.ascontiguousarray(tape)), _p(gZ), _p(gZ0), _p(gU), _p(st), slots_grad,
                                        int(smem_plan), grid)
        if rc != 0:
            raise RuntimeError("the gradient workspace does not fit for this mechanism")
        return gZ0, gU, st
