"""Python wrapper of the CPU oracle (oracle/dojo_oracle.cpp) -- TEST INFRASTRUCTURE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  The product package (dojo.jl_b200) never does.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(_HERE))
import dojo_jl_b200  # noqa: E402,F401
from dojo_jl_b200 import capi  # noqa: E402

LIB_PATH = os.path.join(_HERE, "_build", "libdojo_oracle.so")


def build(force: bool = False) -> str:
    srcs = [os.path.join(_HERE, f) for f in ("dojo_oracle.cpp", "dojo_math.hpp")] + \
           [os.path.join(os.path.dirname(_HERE), "include", "dojo_b200.h")]
    if force or not os.path.exists(LIB_PATH) or any(os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB_PATH)
        L.oracle_create.restype = C.c_void_p
        L.oracle_create.argtypes = [C.POINTER(capi.DojoMechanismDesc)]
        L.oracle_destroy.argtypes = [C.c_void_p]
        for name in ("oracle_num_residual", "oracle_num_input", "oracle_is_tree"):
            getattr(L, name).argtypes = [C.c_void_p]
            getattr(L, name).restype = C.c_int
        dp, ip, vp = capi.c_double_p, capi.c_int32_p, C.c_void_p
        op = C.POINTER(capi.DojoSolverOptions)
        L.oracle_set_solver_mode.argtypes = [vp, C.c_int]
        L.oracle_set_force_iters.argtypes = [vp, C.c_int]
        L.oracle_elimination_order.argtypes = [vp, ip]
        L.oracle_step.argtypes = [vp, op, dp, dp, dp, dp, dp, ip, C.c_uint32]
        L.oracle_step.restype = C.c_int
        L.oracle_step_batch.argtypes = [vp, op, C.c_int, dp, dp, dp, dp, dp, ip, ip, C.c_uint32]
        L.oracle_step_batch_threads.argtypes = [C.POINTER(capi.DojoMechanismDesc), op, C.c_int, dp, dp, dp, ip, ip, C.c_int]
        L.oracle_step_grad_batch_threads.argtypes = [C.POINTER(capi.DojoMechanismDesc), op, C.c_int, dp, dp, dp, dp, dp, ip, ip, C.c_int, C.c_int, C.c_uint32]
        L.oracle_step_grad.argtypes = [vp, op, dp, dp, dp, dp, dp, dp, ip, C.c_uint32, C.c_int]
        L.oracle_step_grad.restype = C.c_int
        L.oracle_set_state.argtypes = [vp, dp, dp, dp]
        L.oracle_set_solution.argtypes = [vp, dp, C.c_double]
        L.oracle_get_solution.argtypes = [vp, dp]
        L.oracle_reset_solution.argtypes = [vp]
        L.oracle_assemble.argtypes = [vp, C.c_double, dp, dp]
        L.oracle_evaluate_rhs.argtypes = [vp, dp, C.c_double, dp]
        L.oracle_violations.argtypes = [vp, dp, dp]
        L.oracle_linear_solve.argtypes = [vp, C.c_int, dp, C.c_int]
        L.oracle_linear_solve.restype = C.c_int
        L.oracle_data_jacobian.argtypes = [vp, dp, C.c_uint32]
        L.oracle_trace.argtypes = [vp, dp, C.c_int]
        L.oracle_trace.restype = C.c_int
        L.oracle_momentum.argtypes = [vp, dp]
        L.oracle_storage_record.argtypes = [vp, dp, dp]
        L.oracle_contact_data_jacobian.argtypes = [vp, dp]
        L.oracle_contact_gradients.argtypes = [vp, dp, C.c_int]
        L.oracle_contact_gradients.restype = C.c_int
        L.oracle_minimal_to_maximal.argtypes = [vp, dp, dp]
        L.oracle_maximal_to_minimal.argtypes = [vp, dp, dp]
        L.oracle_maximal_to_minimal_jacobian.argtypes = [vp, dp, dp]
        L.oracle_minimal_to_maximal_jacobian.argtypes = [vp, dp, dp, C.c_int]
        _lib = L
    return _lib


def _d(a):
    return None if a is None else capi.dptr(a)


class Oracle:
    """One CPU mechanism instance (mutable, single-threaded like the reference's Mechanism)."""

    def __init__(self, mech, opts=None):
        self.mech = mech
        self.L = lib()
        desc, self._keep = capi.flatten(mech)
        self.h = C.c_void_p(self.L.oracle_create(C.byref(desc)))
        self.nres = self.L.oracle_num_residual(self.h)
        self.nu = self.L.oracle_num_input(self.h)
        assert self.nres == mech.nres and self.nu == mech.nu
        self.opts = opts if opts is not None else capi.solver_options()

    def __del__(self):
        try:
            self.L.oracle_destroy(self.h)
        except Exception:
            pass

    # -- step! ---------------------------------------------------------------------------
    def step(self, z, u, fext=None, opts=None, flags=0, return_sol=False):
        z = np.ascontiguousarray(z, dtype=float)
        u = np.ascontiguousarray(u, dtype=float)
        zn = np.empty_like(z)
        sol = np.empty(self.nres)
        it = np.zeros(1, dtype=np.int32)
        st = self.L.oracle_step(self.h, C.byref(opts or self.opts), _d(z), _d(u), _d(fext), _d(zn), _d(sol), capi.iptr(it), flags)
        return (zn, st, int(it[0]), sol) if return_sol else (zn, st, int(it[0]))

    def step_forced(self, z, u, iters, opts=None):
        """step! with EXACTLY `iters` Newton iterations (the convergence test is skipped): the iterate a path reaches when a rounding-level
        flip of the convergence comparison makes it stop one iteration earlier / later than this oracle would."""
        self.L.oracle_set_force_iters(self.h, int(iters))
        try:
            return self.step(z, u, opts=opts)
        finally:
            self.L.oracle_set_force_iters(self.h, -1)

    def step_batch(self, Z, U, opts=None, flags=0):
        """Z [B x 13Nb], U [B x nu] (row = environment, i.e. the column-major [feature x B] buffer)."""
        Z = np.ascontiguousarray(Z, dtype=float)
        U = np.ascontiguousarray(U, dtype=float)
        B = Z.shape[0]
        Zn = np.empty_like(Z)
        st = np.zeros(B, dtype=np.int32)
        it = np.zeros(B, dtype=np.int32)
        self.L.oracle_step_batch(self.h, C.byref(opts or self.opts), B, _d(Z), _d(U), None, _d(Zn), None, capi.iptr(st), capi.iptr(it), flags)
        return Zn, st, it

    def step_grad(self, z, u, opts=None, use_factor=False, flags=0):
        z = np.ascontiguousarray(z, dtype=float)
        u = np.ascontiguousarray(u, dtype=float)
        ns = 12 * self.mech.Nb
        zn = np.empty_like(z)
        Fz = np.empty((ns, ns), order="F")
        Fu = np.empty((ns, self.nu), order="F")
        it = np.zeros(1, dtype=np.int32)
        st = self.L.oracle_step_grad(self.h, C.byref(opts or self.opts), _d(z), _d(u), None, _d(zn),
                                     Fz.ctypes.data_as(capi.c_double_p), Fu.ctypes.data_as(capi.c_double_p), capi.iptr(it), flags, int(use_factor))
        return zn, Fz, Fu, st, int(it[0])

    def contact_data_jacobian(self):
        """data Jacobian restricted to the contact data columns (gradients/data.jl:152-192): [nres, 5 Ni]"""
        out = np.empty((self.nres, 5 * self.mech.Ni))
        self.L.oracle_contact_data_jacobian(self.h, _d(out))
        return out

    def contact_gradients(self, use_factor=False):
        """get_contact_gradients (gradients/contact.jl:1-55) at the solution of the last step: d z' / d theta, theta = per contact
        [friction_coefficient, contact_radius, contact_origin(3)]; [12 Nb, 5 Ni]."""
        Fc = np.empty((12 * self.mech.Nb, 5 * self.mech.Ni), order="F")
        rc = self.L.oracle_contact_gradients(self.h, Fc.ctypes.data_as(capi.c_double_p), int(use_factor))
        if rc != 0:
            raise np.linalg.LinAlgError("singular KKT matrix")
        return Fc

    # -- pieces for the property tests -----------------------------------------------------
    def set_state(self, z, u=None, fext=None):
        z = np.ascontiguousarray(z, dtype=float)
        u = np.zeros(self.nu) if u is None else np.ascontiguousarray(u, dtype=float)
        self.L.oracle_set_state(self.h, _d(z), _d(u), _d(fext))

    def set_solution(self, sol, mu=0.0):
        sol = np.ascontiguousarray(sol, dtype=float)
        self.L.oracle_set_solution(self.h, _d(sol), float(mu))

    def get_solution(self):
        sol = np.empty(self.nres)
        self.L.oracle_get_solution(self.h, _d(sol))
        return sol

    def reset_solution(self):
        self.L.oracle_reset_solution(self.h)

    def assemble(self, mu=0.0):
        A = np.empty((self.nres, self.nres))
        b = np.empty(self.nres)
        self.L.oracle_assemble(self.h, float(mu), _d(A), _d(b))
        return A, b

    def evaluate_rhs(self, sol, mu=0.0):
        sol = np.ascontiguousarray(sol, dtype=float)
        out = np.empty(self.nres)
        self.L.oracle_evaluate_rhs(self.h, _d(sol), float(mu), _d(out))
        return out

    # minimal <-> maximal coordinate maps (mechanism/state.jl:9-66)
    @property
    def nmin(self):
        return 2 * self.nu

    def minimal_to_maximal(self, x):
        x = np.ascontiguousarray(x, dtype=float)
        z = np.empty(13 * self.mech.Nb)
        self.L.oracle_minimal_to_maximal(self.h, _d(x), _d(z))
        return z

    def maximal_to_minimal(self, z):
        z = np.ascontiguousarray(z, dtype=float)
        x = np.empty(self.nmin)
        self.L.oracle_maximal_to_minimal(self.h, _d(z), _d(x))
        return x

    # Jacobians of the maps (gradients/state.jl:9-56, :136-179) and the minimal-coordinate gradients (:192-217)
    def maximal_to_minimal_jacobian(self, z):
        """(2 nu) x (12 Nb): d(minimal state) / d(maximal state, attitude-reduced [x, v, phi, w] per body)."""
        z = np.ascontiguousarray(z, dtype=float)
        J = np.empty((self.nmin, 12 * self.mech.Nb), order="F")
        self.L.oracle_maximal_to_minimal_jacobian(self.h, _d(z), J.ctypes.data_as(capi.c_double_p))
        return J

    def minimal_to_maximal_jacobian(self, z, body_order_literal=False):
        """(12 Nb) x (2 nu) at the maximal state z (the reference evaluates at the mechanism's stored state)."""
        z = np.ascontiguousarray(z, dtype=float)
        J = np.empty((12 * self.mech.Nb, self.nmin), order="F")
        self.L.oracle_minimal_to_maximal_jacobian(self.h, _d(z), J.ctypes.data_as(capi.c_double_p), int(body_order_literal))
        return J

    def minimal_gradients(self, x, u, opts=None):
        """get_minimal_gradients! (gradients/state.jl:192-217), consistent variant (SURVEY Q2): the maximal gradients
        and minimal_to_maximal_jacobian at z = minimal_to_maximal(x), maximal_to_minimal_jacobian at the true next state.
        Returns (x_next, dx'/dx [2nu x 2nu], dx'/du [2nu x nu], status, iters)."""
        z = self.minimal_to_maximal(x)
        zn, Fz, Fu, st, it = self.step_grad(z, u, opts=opts)
        M = self.maximal_to_minimal_jacobian(zn)
        N = self.minimal_to_maximal_jacobian(z)
        return self.maximal_to_minimal(zn), M @ Fz @ N, M @ Fu, st, it

    def violations(self):
        r, b = C.c_double(), C.c_double()
        self.L.oracle_violations(self.h, C.byref(r), C.byref(b))
        return r.value, b.value

    def linear_solve(self, b, mode=0):
        x = np.array(b, dtype=float, order="C", copy=True)
        m = 1 if x.ndim == 1 else x.shape[1]
        rc = self.L.oracle_linear_solve(self.h, mode, _d(x), m)
        if rc != 0:
            raise np.linalg.LinAlgError("singular block")
        return x

    def data_jacobian(self, flags=0):
        """d(rhs)/d[state, input] at the current state, input and solution; flags: DOJO_FLAG_Q17_LITERAL_INPUT_JACOBIAN omits the
        inputs' configuration derivative as the reference's gradients/data.jl does."""
        out = np.empty((self.nres, 12 * self.mech.Nb + self.nu))
        self.L.oracle_data_jacobian(self.h, _d(out), int(flags))
        return out

    def trace(self):
        buf = np.empty(4 * 64)
        n = self.L.oracle_trace(self.h, _d(buf), buf.size)
        return buf[: 4 * n].reshape(n, 4)

    def elimination_order(self):
        out = np.zeros(self.mech.Ne + self.mech.Nb + self.mech.Ni, dtype=np.int32)
        self.L.oracle_elimination_order(self.h, capi.iptr(out))
        return out

    def set_solver_mode(self, mode):
        self.L.oracle_set_solver_mode(self.h, mode)

    def storage_record(self):
        """save_to_storage! after the last step's solve: (per body [px; pq; vl; wl] as [Nb, 12],
        [p_linear(3); p_angular(3); kinetic; potential])  (simulation/storage.jl:50-67, mechanics/{momentum,energy}.jl)."""
        body = np.empty((self.mech.Nb, 12))
        diag = np.empty(8)
        self.L.oracle_storage_record(self.h, _d(body), _d(diag))
        return body, diag

    def momentum(self):
        """[p_linear; p_angular] right after the last step's solve (mechanics/momentum.jl:17-86)."""
        out = np.empty(6)
        self.L.oracle_momentum(self.h, _d(out))
        return out


def step_batch_threads(mech, Z, U, opts=None, nthreads=1):
    """Step a batch on `nthreads` C++ threads (one mechanism instance each).  Returns (Zn, status, iters)."""
    L = lib()
    desc, keep = capi.flatten(mech)
    Z = np.ascontiguousarray(Z, dtype=float)
    U = np.ascontiguousarray(U, dtype=float)
    B = Z.shape[0]
    Zn = np.empty_like(Z)
    st = np.zeros(B, dtype=np.int32)
    it = np.zeros(B, dtype=np.int32)
    o = opts if opts is not None else capi.solver_options()
    L.oracle_step_batch_threads(C.byref(desc), C.byref(o), B, _d(Z), _d(U), _d(Zn), capi.iptr(st), capi.iptr(it), int(nthreads))
    return Zn, st, it


def step_grad_batch_threads(mech, Z, U, opts=None, nthreads=1, keep=False, use_factor=False, flags=0):
    """step! + get_maximal_gradients for a batch on `nthreads` C++ threads.  keep=False drops the Jacobians (timing only).
    Returns (Zn, status, iters[, Fz [B, 12Nb, 12Nb] column-major per environment, Fu])."""
    L = lib()
    desc, _keep = capi.flatten(mech)
    Z = np.ascontiguousarray(Z, dtype=float)
    U = np.ascontiguousarray(U, dtype=float)
    B = Z.shape[0]
    ns = 12 * mech.Nb
    Zn = np.empty_like(Z)
    st = np.zeros(B, dtype=np.int32)
    it = np.zeros(B, dtype=np.int32)
    Fz = np.empty((B, ns, ns)) if keep else None
    Fu = np.empty((B, mech.nu, ns)) if keep else None
    o = opts if opts is not None else capi.solver_options()
    L.oracle_step_grad_batch_threads(C.byref(desc), C.byref(o), B, _d(Z), _d(U), _d(Zn), _d(Fz), _d(Fu), capi.iptr(st), capi.iptr(it), int(nthreads),
                                     int(use_factor), int(flags))
    return (Zn, st, it, Fz, Fu) if keep else (Zn, st, it)
