"""The closed-loop rollout on the CPU -- TEST INFRASTRUCTURE for tests/test_rollout_feedback.py.

FeedbackEmu runs the closed-loop rollout dojo_step_kernel<false, false, false, false, false, FB = true> on CPU fibers, as
dojo_rollout_feedback does, and also returns the kernel's scratch of minimal states (x_t of every environment's last step).  Its entry
point, hostemu_rollout_feedback, is appended here to the emulation's generated translation unit (gen.generate(): the product's kernel,
handle and table builder with driver.inc), which is compiled into a library of its own.  So FeedbackEmu has every entry point of HostEmu
plus this one, and its open-loop rollouts (step) run in the same library as its closed-loop ones."""
import contextlib
import ctypes as C
import os
import subprocess

import numpy as np

from dojo_jl_b200 import capi
from dojo_jl_b200.solver import feedback_arrays
from . import gen
from .harness import HostEmu, _p, _vp, _ip

ENTRY = r"""
// dojo_rollout_feedback: the closed-loop rollout kernel (FB) with the law's arrays as DojoFeedback holds them (host arrays here).  Ua nullable
// (then u_t goes to a [nu x B] scratch, as in the library); x [2nu x B] is the kernel's x scratch: on return, x_t of each environment's last step
extern "C" int hostemu_rollout_feedback(void* p, const DojoSolverOptions* opts, int B, int T, const double* Z0, const DojoFeedback* fb, double* xi, double* Zf,
                                        double* traj, double* Ua, int32_t* status, double* x, int slots, int smem_plan, int grid) {
  DojoHandle* h = static_cast<EmuHandle*>(p)->h;
  std::vector<double> u((size_t)B * h->plan.nu);
  int counter = 0;
  StepArgs a = emu_args(h, opts, B, false, slots, smem_plan != 0, &counter);
  a.Z = Z0; a.Zn = Zf; a.status = status; a.T = T; a.traj = traj;
  a.fb_K = fb->K; a.fb_Ki = fb->K_i; a.fb_xref = fb->x_ref; a.fb_uref = fb->u_ref; a.fb_steps = fb->steps; a.fb_envs = fb->envs;
  a.fb_x = x; a.fb_xi = xi; a.fb_u = Ua ? Ua : u.data(); a.fb_u_T = Ua ? 1 : 0;
  emu_launch<false, false, false, false, false, true>(h, a, grid, slots, smem_plan != 0);
  return 0;
}
"""


def build() -> str:
    """the emulation library with hostemu_rollout_feedback, in a directory of its own next to gen.build()'s (same compiler flags)"""
    d = os.path.join(gen.build_dir(), "feedback")
    os.makedirs(d, exist_ok=True)
    lib = os.path.join(d, "libdojo_hostemu_feedback_fma.so" if gen.FMA else "libdojo_hostemu_feedback.so")
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


@contextlib.contextmanager
def _patched(obj, name, value):
    old = getattr(obj, name)
    setattr(obj, name, value)
    try:
        yield
    finally:
        setattr(obj, name, old)


class FeedbackEmu(HostEmu):
    """HostEmu's kernels (step, step_grad, kinjac) and the closed-loop rollout (rollout_feedback), all from the library of build()."""

    def __init__(self, mech):
        lib = build()
        with _patched(gen, "build", lambda: lib):  # HostEmu loads gen.build()'s library; this one is a superset of it
            super().__init__(mech)
        self.L.hostemu_rollout_feedback.argtypes = [_vp, C.POINTER(capi.DojoSolverOptions), _ip, _ip, _vp, C.POINTER(capi.DojoFeedback), _vp, _vp,
                                                    _vp, _vp, _vp, _vp, _ip, _ip, _ip]

    def rollout_feedback(self, Z0, T, K, x_ref=None, u_ref=None, K_i=None, xi=None, opts=None, slots=2, smem_plan=True, grid=2, applied=True):
        """dojo_rollout_feedback with BatchedStepper.rollout_feedback's argument shapes.  Returns (Z_final [B, nz], status_any [B],
        Z_traj [T, B, nz], U_applied [T, B, nu] (None with applied=False: the kernel writes u_t to a scratch), xi [B, 2nu] or None,
        x [B, 2nu] = x_{T-1})."""
        Z0 = np.ascontiguousarray(np.atleast_2d(Z0), dtype=np.float64)
        B, nu = Z0.shape[0], self.mech.nu
        steps, envs, Kc, xr, ur, Kic = feedback_arrays(T, B, nu, K, x_ref, u_ref, K_i)
        fb = capi.DojoFeedback(steps, envs, capi.dptr(Kc), None if Kic is None else capi.dptr(Kic), None if xr is None else capi.dptr(xr),
                               None if ur is None else capi.dptr(ur))
        xi = None if Kic is None else (np.zeros((B, 2 * nu)) if xi is None else np.array(np.broadcast_to(np.asarray(xi, dtype=np.float64), (B, 2 * nu))))
        Zf, traj = np.empty_like(Z0), np.empty((T, B, Z0.shape[1]))
        Ua = np.empty((T, B, nu)) if applied else None
        st, x = np.zeros(B, dtype=np.int32), np.full((B, 2 * nu), np.nan)
        o = opts if opts is not None else capi.solver_options()
        self.L.hostemu_rollout_feedback(self.h, C.byref(o), B, T, _p(Z0), C.byref(fb), _p(xi), _p(Zf), _p(traj), _p(Ua), _p(st), _p(x), slots,
                                        int(smem_plan), grid)
        return Zf, st, traj, Ua, xi, x
