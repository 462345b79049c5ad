"""ctypes wrapper of the host emulation of the step / gradient kernels -- TEST INFRASTRUCTURE (see cuda_shim.h, gen.py)."""
import ctypes as C

import numpy as np

from dojo_jl_b200 import capi
from . import gen

_vp, _ip = C.c_void_p, C.c_int


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


class HostEmu:
    """The product's dojo_step_kernel<false/true> run on CPU fibers for one mechanism.  The ctypes signatures of every entry point of
    driver.inc are declared here, also those that only the subclasses in trace.py, small.py and rollout_grad.py call."""

    def __init__(self, mech):
        L = C.CDLL(gen.build())
        L.hostemu_create.restype = _vp
        L.hostemu_create.argtypes = [C.POINTER(capi.DojoMechanismDesc)]
        L.hostemu_destroy.argtypes = [_vp]
        L.hostemu_last_error.restype = C.c_char_p
        for n in ("hostemu_num_residual", "hostemu_num_input", "hostemu_warps_per_env"):
            getattr(L, n).argtypes = [_vp]
        L.hostemu_arena_bytes.argtypes = [_vp, _ip]
        L.hostemu_arena_bytes.restype = C.c_long
        op = C.POINTER(capi.DojoSolverOptions)
        L.hostemu_step.argtypes = [_vp, op, _ip, _ip, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint32, _ip, _ip, _ip, _vp]
        L.hostemu_step_grad.argtypes = [_vp, op, _ip, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ip, _ip, _ip, _ip, _vp]
        L.hostemu_kinjac.argtypes = [_vp, _ip, _ip, _ip, _vp, _vp, _vp, _vp, _vp, _vp]
        L.hostemu_step_trace.argtypes = [_vp, op, _ip, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint32, _ip, _ip, _ip]
        L.hostemu_step_small.argtypes = [_vp, op, _ip, _ip, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint32, _ip, _ip, _vp]
        L.hostemu_small_step_ok.argtypes = [_vp, _ip]
        L.hostemu_rollout_grad.argtypes = [_vp, op, _ip, _ip, _vp, _vp, _vp, _vp, _vp, _vp, _ip, _ip, _ip, _ip]
        self.L, self.mech = L, mech
        desc, self._keep = capi.flatten(mech)
        h = L.hostemu_create(C.byref(desc))
        if not h:
            raise RuntimeError("hostemu_create failed: " + L.hostemu_last_error().decode())
        self.h = C.c_void_p(h)
        assert L.hostemu_num_residual(self.h) == mech.nres and L.hostemu_num_input(self.h) == mech.nu

    def __del__(self):
        try:
            self.L.hostemu_destroy(self.h)
        except Exception:
            pass

    def step(self, Z, U=None, opts=None, T=1, fext=None, flags=0, slots=1, smem_plan=True, grid=1, record=False):
        """dojo_step (T = 1) / dojo_rollout (T > 1, U [T, B, nu]).  Returns (Z_next, status, iters, sol[, traj])."""
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=np.float64)
        B = Z.shape[0]
        if U is not None:
            U = np.ascontiguousarray(U, dtype=np.float64)
        Zn = np.empty_like(Z)
        sol = np.empty((B, self.mech.nres))
        st, it = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        traj = np.empty((T, B, Z.shape[1])) if record else None
        o = opts if opts is not None else capi.solver_options()
        self.L.hostemu_step(self.h, C.byref(o), B, T, _p(Z), _p(U), _p(fext), _p(Zn), _p(sol), _p(st), _p(it), flags, slots, int(smem_plan), grid, _p(traj))
        return (Zn, st, it, sol, traj) if record else (Zn, st, it, sol)

    def step_gather(self, Z, U, rank, bufs, flags, slots=2, grid=2, opts=None):
        """dojo_step_gather_async for one rank: bufs[r] = gathered buffer of rank r [world * B, nz], flags[r] = its counter (uint64[1])."""
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=np.float64)
        U = np.ascontiguousarray(U, dtype=np.float64)
        B, world = Z.shape[0], len(bufs)
        Zn = np.empty_like(Z)
        st, it = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        pb = (C.c_void_p * world)(*[b.ctypes.data for b in bufs])
        pf = (C.c_void_p * world)(*[f.ctypes.data for f in flags])
        o = opts if opts is not None else capi.solver_options()
        self.L.hostemu_step_gather.argtypes = [_vp, C.POINTER(capi.DojoSolverOptions), _ip, _vp, _vp, _vp, _vp, _vp, _ip, _ip, _vp, _vp, _ip, _ip]
        rc = self.L.hostemu_step_gather(self.h, C.byref(o), B, _p(Z), _p(U), _p(Zn), _p(st), _p(it), world, rank, pb, pf, slots, grid)
        assert rc == 0
        return Zn, st, it

    def step_grad(self, Z, U=None, opts=None, slots=1, slots_grad=1, smem_plan=True, publish_order=True, contact=False, flags=0):
        """dojo_step_grad (contact=True: dojo_step_grad_contact).  Returns (Z_next, Fz [B, 12Nb, 12Nb], Fu [B, 12Nb, nu][, Fc [B, 12Nb, 5Ni]],
        status, iters)."""
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=np.float64)
        B = Z.shape[0]
        U = np.zeros((B, self.mech.nu)) if U is None else np.ascontiguousarray(U, dtype=np.float64)
        ng = 12 * self.mech.Nb
        Zn = np.empty_like(Z)
        Fz, Fu = np.empty((B, ng, ng)), np.empty((B, self.mech.nu, ng))
        st, it = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        Fc = np.empty((B, 5 * self.mech.Ni, ng)) if contact else None
        self.L.hostemu_set_grad_flags(C.c_uint32(flags))
        rc = self.L.hostemu_step_grad(self.h, C.byref(o), B, _p(Z), _p(U), _p(Zn), _p(Fz), _p(Fu), _p(st), _p(it), slots, slots_grad, int(smem_plan),
                                      int(publish_order), _p(Fc))
        if rc != 0:
            self.L.hostemu_set_grad_flags(C.c_uint32(0))
            raise RuntimeError("the gradient workspace does not fit for this mechanism")
        self.L.hostemu_set_grad_flags(C.c_uint32(0))
        if contact:
            return Zn, Fz.transpose(0, 2, 1), Fu.transpose(0, 2, 1), Fc.transpose(0, 2, 1), st, it
        return Zn, Fz.transpose(0, 2, 1), Fu.transpose(0, 2, 1), st, it

    def kinjac(self, mode, Z, Zn=None, Fz=None, Fu=None, grid=2):
        """dojo_kinjac_kernel with 128-thread CTAs.  mode 0: M [B, 2nu, 12Nb]; 1: N [B, 12Nb, 2nu]; 2: (Gx, Gu) from Fz / Fu in
        math layout [B, 12Nb, 12Nb] / [B, 12Nb, nu]."""
        m = self.mech
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=np.float64)
        B, nm, ns = Z.shape[0], 2 * m.nu, 12 * m.Nb
        if mode == 0:
            J = np.empty((B, ns, nm))
            self.L.hostemu_kinjac(self.h, 0, B, grid, _p(Z), None, None, None, _p(J), None)
            return J.transpose(0, 2, 1)
        if mode == 1:
            J = np.empty((B, nm, ns))
            self.L.hostemu_kinjac(self.h, 1, B, grid, _p(Z), None, None, None, _p(J), None)
            return J.transpose(0, 2, 1)
        Zn = np.ascontiguousarray(np.atleast_2d(Zn), dtype=np.float64)
        Fzc = np.ascontiguousarray(np.asarray(Fz, dtype=np.float64).transpose(0, 2, 1))
        Fuc = np.ascontiguousarray(np.asarray(Fu, dtype=np.float64).transpose(0, 2, 1))
        Gx, Gu = np.empty((B, nm, nm)), np.empty((B, m.nu, nm))
        self.L.hostemu_kinjac(self.h, 2, B, grid, _p(Z), _p(Zn), _p(Fzc), _p(Fuc), _p(Gx), _p(Gu))
        return Gx.transpose(0, 2, 1), Gu.transpose(0, 2, 1)
