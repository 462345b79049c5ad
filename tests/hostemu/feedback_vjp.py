"""Reverse mode through a closed-loop rollout on the CPU -- TEST INFRASTRUCTURE for tests/test_rollout_feedback_vjp.py.

FeedbackVjpEmu runs, on CPU fibers, the two launches of dojo_rollout_feedback_tape / dojo_rollout_feedback_vjp: the closed-loop tape
dojo_step_kernel<false, ..., REC = true, FB = true> and its adjoint dojo_step_kernel<true, ..., FB = true, VJP = true>.  Their entry points
are appended, with those of feedback.py and vjp.py, to the emulation's generated translation unit (gen.generate(): the product's kernel,
handle and table builder with driver.inc), which is compiled into a library of its own.  So FeedbackVjpEmu also has the open-loop tape /
adjoint, the closed-loop rollout, rollout_grad and the map Jacobians of HostEmu, all from the same library.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from dojo_jl_b200 import capi
from dojo_jl_b200.solver import feedback_arrays
from . import feedback, gen, vjp
from .feedback import FeedbackEmu, _patched
from .harness import _ip, _p, _vp
from .rollout_grad import RolloutGradEmu

ENTRY = r"""
// dojo_rollout_feedback_tape: the closed-loop tape (REC + FB).  traj [nz x B x (T + 1)] holds Z0 in slab 0
extern "C" int hostemu_rollout_feedback_tape(void* p, const DojoSolverOptions* opts, int B, int T, double* traj, const DojoFeedback* fb, double* xi,
                                             double* X, double* Xi, double* Ua, double* tape, int32_t* status, int32_t* iters, int slots, int smem_plan,
                                             int grid) {
  DojoHandle* h = static_cast<EmuHandle*>(p)->h;
  int counter = 0;
  StepArgs a = emu_args(h, opts, B, false, slots, smem_plan != 0, &counter);
  a.Z = traj; a.traj = traj + (size_t)B * h->plan.nz; a.T = T; a.sol_raw = tape; a.status = status; a.iters = iters;
  a.fb_K = fb->K; a.fb_Ki = fb->K_i; a.fb_xref = fb->x_ref; a.fb_uref = fb->u_ref; a.fb_steps = fb->steps; a.fb_envs = fb->envs;
  a.fb_xi = xi; a.fb_u = Ua; a.fb_u_T = 1; a.fb_xtraj = X; a.fb_xitraj = Xi;
  emu_launch<false, false, false, false, true, true>(h, a, grid, slots, smem_plan != 0);
  return 0;
}
// dojo_rollout_feedback_vjp: the closed-loop adjoint (VJP + FB) in the gradient launch configuration
extern "C" int hostemu_rollout_feedback_vjp(void* p, int B, int T, const DojoFeedback* fb, const double* traj, const double* X, const double* Xi,
                                            const double* Ua, const double* tape, const double* gZ, const double* gX, const double* gUa,
                                            const DojoFeedbackGrad* out, double* gZ0, double* gxi0, int32_t* status, int slots_grad, int smem_plan,
                                            int grid) {
  DojoHandle* h = static_cast<EmuHandle*>(p)->h;
  if (!h->grad_bytes) return -1;
  std::vector<double> ws((4 * (size_t)h->plan.nu + 12 * (size_t)h->plan.Nb) * B);
  int counter = 0;
  StepArgs g = emu_args(h, nullptr, B, true, slots_grad, smem_plan != 0, &counter);
  g.Z = traj; g.U = Ua; g.sol_raw = const_cast<double*>(tape); g.status = status; g.T = T;
  g.vjp_gZ = gZ; g.vjp_lam = gZ0;
  g.fb_K = fb->K; g.fb_Ki = fb->K_i; g.fb_xref = fb->x_ref; g.fb_uref = fb->u_ref; g.fb_steps = fb->steps; g.fb_envs = fb->envs; g.fb_xi = gxi0;
  g.fb_xtraj = const_cast<double*>(X); g.fb_xitraj = const_cast<double*>(Xi); g.fbv_gX = gX; g.fbv_gUa = gUa;
  g.fbv_gK = out->K; g.fbv_gKi = out->K_i; g.fbv_gxref = out->x_ref; g.fbv_guref = out->u_ref; g.fbv_ws = ws.data();
  if (smem_plan) emu_launch<true, true, false, false, false, true, true>(h, g, grid, slots_grad, true);
  else emu_launch<true, false, false, false, false, true, true>(h, g, grid, slots_grad, false);
  return 0;
}
"""


def build() -> str:
    """the emulation library with the closed-loop, tape and adjoint entry points, in a directory of its own (same compiler flags)"""
    d = os.path.join(gen.build_dir(), "feedback_vjp")
    os.makedirs(d, exist_ok=True)
    lib = os.path.join(d, "libdojo_hostemu_feedback_vjp_fma.so" if gen.FMA else "libdojo_hostemu_feedback_vjp.so")
    if not gen.stale(lib, gen.DEPS + [os.path.abspath(__file__), os.path.abspath(feedback.__file__), os.path.abspath(vjp.__file__)]):
        return lib
    with _patched(gen, "build_dir", lambda: d):  # generate() writes its TU into d, not over the one gen.build() compiles
        tu = gen.generate()
    with open(tu, "a") as f:
        f.write(feedback.ENTRY + vjp.ENTRY + ENTRY)
    fp = ["-ffp-contract=fast", "-march=x86-64-v3"] if gen.FMA else ["-ffp-contract=off"]
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared"] + fp + ["-Wno-unknown-pragmas", "-Wno-unused-function",
                           "-Wno-unused-variable", "-Wno-unused-but-set-variable", "-o", lib + ".tmp", tu])
    os.replace(lib + ".tmp", lib)
    return lib


def law(m, T, B, K, x_ref=None, u_ref=None, K_i=None):
    """(DojoFeedback, arrays kept alive, (steps, envs)) from BatchedStepper.rollout_feedback's argument shapes"""
    steps, envs, Kc, xr, ur, Kic = feedback_arrays(T, B, m.nu, K, x_ref, u_ref, K_i)
    fb = capi.DojoFeedback(steps, envs, capi.dptr(Kc), None if Kic is None else capi.dptr(Kic), None if xr is None else capi.dptr(xr),
                           None if ur is None else capi.dptr(ur))
    return fb, (Kc, xr, ur, Kic), (steps, envs)


class FeedbackVjpEmu(RolloutGradEmu):
    """HostEmu's kernels, rollout_grad, the closed-loop rollout, the open-loop tape / adjoint and the closed-loop tape / adjoint."""

    rollout_feedback = FeedbackEmu.rollout_feedback
    rollout_tape = vjp.VjpEmu.rollout_tape
    rollout_vjp = vjp.VjpEmu.rollout_vjp

    def __init__(self, mech):
        lib = build()
        with _patched(gen, "build", lambda: lib):  # HostEmu loads gen.build()'s library; this one is a superset of it
            super().__init__(mech)
        op = C.POINTER(capi.DojoSolverOptions)
        fp = C.POINTER(capi.DojoFeedback)
        self.L.hostemu_rollout_feedback.argtypes = [_vp, op, _ip, _ip, _vp, fp, _vp, _vp, _vp, _vp, _vp, _vp, _ip, _ip, _ip]
        self.L.hostemu_rollout_tape.argtypes = [_vp, op, _ip, _ip, _vp, _vp, _vp, _vp, _vp, _ip, _ip, _ip]
        self.L.hostemu_rollout_vjp.argtypes = [_vp, _ip, _ip, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ip, _ip, _ip]
        self.L.hostemu_rollout_feedback_tape.argtypes = [_vp, op, _ip, _ip, _vp, fp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ip, _ip, _ip]
        self.L.hostemu_rollout_feedback_vjp.argtypes = [_vp, _ip, _ip, fp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(capi.DojoFeedbackGrad),
                                                        _vp, _vp, _vp, _ip, _ip, _ip]

    def rollout_feedback_tape(self, Z0, T, K, x_ref=None, u_ref=None, K_i=None, xi=None, opts=None, slots=2, smem_plan=True, grid=2):
        """dojo_rollout_feedback_tape.  Returns a dict: Z_traj [T+1, B, nz], X_traj [T+1, B, 2nu], Xi_traj [T, B, 2nu] or None, U [T, B, nu],
        tape [T, B, nres], status / iters [T, B], xi [B, 2nu] (after the call) or None."""
        m = self.mech
        Z0 = np.ascontiguousarray(np.atleast_2d(Z0), dtype=np.float64)
        B, nx = Z0.shape[0], 2 * m.nu
        fb, keep, _ = law(m, T, B, K, x_ref, u_ref, K_i)
        xi = None if K_i is None else (np.zeros((B, nx)) if xi is None else np.array(np.broadcast_to(np.asarray(xi, dtype=np.float64), (B, nx))))
        traj = np.empty((T + 1, B, m.nz))
        traj[0] = Z0
        X, Xi = np.full((T + 1, B, nx), np.nan), (None if K_i is None else np.full((T, B, nx), np.nan))
        Ua, tape = np.empty((T, B, m.nu)), np.empty((T, B, m.nres))
        st, it = np.zeros((T, B), dtype=np.int32), np.zeros((T, B), dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        self.L.hostemu_rollout_feedback_tape(self.h, C.byref(o), B, T, _p(traj), C.byref(fb), _p(xi), _p(X), _p(Xi), _p(Ua), _p(tape), _p(st), _p(it),
                                             slots, int(smem_plan), grid)
        return dict(Z_traj=traj, X_traj=X, Xi_traj=Xi, U=Ua, tape=tape, status=st, iters=it, xi=xi)

    def rollout_feedback_vjp(self, rec, K, x_ref=None, u_ref=None, K_i=None, gZ=None, gX=None, gUa=None, slots_grad=1, smem_plan=True, grid=1,
                             outputs=("K", "K_i", "x_ref", "u_ref")):
        """dojo_rollout_feedback_vjp on the record `rec` of rollout_feedback_tape.  Returns a dict: gZ0 [B, 12Nb], gxi0 [B, 2nu] or None,
        status [B], and per requested output the kernel's per-environment array [steps, B, ...] (K / K_i as [steps, B, nu, 2nu])."""
        m = self.mech
        T, B = rec["tape"].shape[:2]
        nu, nx, ng = m.nu, 2 * m.nu, 12 * m.Nb
        fb, keep, (steps, _) = law(m, T, B, K, x_ref, u_ref, K_i)
        shapes = {"K": (steps, B, nx, nu), "K_i": (steps, B, nx, nu), "x_ref": (steps, B, nx), "u_ref": (steps, B, nu)}
        outs = {k: np.full(shapes[k], -7.0) for k in outputs if not (k == "K_i" and K_i is None)}
        g = capi.DojoFeedbackGrad(*[capi.dptr(outs[k]) if k in outs else None for k in ("K", "K_i", "x_ref", "u_ref")])
        c = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)  # noqa: E731
        gZ, gX, gUa = c(gZ), c(gX), c(gUa)
        assert gZ is None or gZ.shape == (T + 1, B, ng)
        assert gX is None or gX.shape == (T + 1, B, nx)
        assert gUa is None or gUa.shape == (T, B, nu)
        gZ0 = np.full((B, ng), -7.0)
        gxi0 = None if K_i is None else np.full((B, nx), -7.0)
        st = np.full(B, -1, dtype=np.int32)
        rc = self.L.hostemu_rollout_feedback_vjp(self.h, B, T, C.byref(fb), _p(c(rec["Z_traj"])), _p(c(rec["X_traj"])), _p(c(rec["Xi_traj"])),
                                                 _p(c(rec["U"])), _p(c(rec["tape"])), _p(gZ), _p(gX), _p(gUa), C.byref(g), _p(gZ0), _p(gxi0), _p(st),
                                                 slots_grad, int(smem_plan), grid)
        if rc != 0:
            raise RuntimeError("the gradient workspace does not fit for this mechanism")
        res = dict(gZ0=gZ0, gxi0=gxi0, status=st)
        for k, v in outs.items():
            res[k] = v.swapaxes(-1, -2) if v.ndim == 4 else v
        return res
