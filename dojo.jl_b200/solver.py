"""ctypes binding of the product library libdojo_b200.so (include/dojo_b200.h).

This is the ONLY compute path of the package: if the CUDA library is missing or no CUDA device is
present, construction fails loudly (RuntimeError) -- there is no CPU fallback.
"""
import ctypes as C
import os
from typing import Optional

import numpy as np

from . import capi
from .mechanism import Mechanism

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdojo_b200.so")

DOJO_FLAG_Q1_LITERAL_RETURN = 1
DOJO_FLAG_Q2_LITERAL_GRADIENTS = 2  # get_maximal_gradients! literally: data Jacobian after update_state! (include/dojo_b200.h)
DOJO_FLAG_Q17_LITERAL_INPUT_JACOBIAN = 4  # data Jacobian without d(input impulse)/d(configuration), as gradients/data.jl (include/dojo_b200.h)
STATUS = {0: "success", 1: "failed", 2: "excessive_angular_velocity", 3: "nonfinite"}

EXPORTS = ["dojo_default_options", "dojo_create", "dojo_destroy", "dojo_last_error", "dojo_num_state", "dojo_num_input",
           "dojo_num_residual", "dojo_num_grad_state", "dojo_shared_bytes_per_env", "dojo_step", "dojo_step_async",
           "dojo_step_grad", "dojo_step_grad_async", "dojo_rollout", "dojo_rollout_async", "dojo_launch_count",
           "dojo_num_minimal", "dojo_minimal_to_maximal", "dojo_maximal_to_minimal", "dojo_minimal_to_maximal_async",
           "dojo_maximal_to_minimal_async", "dojo_step_minimal", "dojo_step_minimal_flags", "dojo_maximal_to_minimal_jacobian", "dojo_minimal_to_maximal_jacobian",
           "dojo_maximal_to_minimal_jacobian_async", "dojo_minimal_to_maximal_jacobian_async", "dojo_minimal_gradients", "dojo_env_num_state", "dojo_env_num_action", "dojo_env_step",
           "dojo_env_step_async", "dojo_env_reset", "dojo_env_rollout", "dojo_env_policy_rollout", "dojo_update_params", "dojo_num_contact_data", "dojo_step_grad_contact",
           "dojo_step_grad_contact_async", "dojo_step_record", "dojo_step_record_async", "dojo_simulate_record",
           "dojo_gather_create", "dojo_gather_export", "dojo_gather_connect", "dojo_gather_buffer", "dojo_gather_destroy", "dojo_step_gather_async",
           "dojo_step_grad_gather_async", "dojo_step_trace", "dojo_step_trace_async", "dojo_rollout_grad", "dojo_rollout_grad_async",
           "dojo_rollout_minimal_gradients", "dojo_rollout_feedback", "dojo_rollout_feedback_async", "dojo_lqr_backward", "dojo_lqr_backward_async"]

_lib = None


def load_library():
    """Load libdojo_b200.so (built in-tree by build.py).  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(nvcc, sm_90a).  dojo.jl_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    dp, ip, vp = capi.c_double_p, capi.c_int32_p, C.c_void_p
    op = C.POINTER(capi.DojoSolverOptions)
    L.dojo_default_options.argtypes = [op]
    L.dojo_create.argtypes = [C.POINTER(capi.DojoMechanismDesc), C.c_int, C.c_int, C.POINTER(vp)]
    L.dojo_create.restype = C.c_int
    L.dojo_destroy.argtypes = [vp]
    L.dojo_last_error.argtypes = [vp]
    L.dojo_last_error.restype = C.c_char_p
    for n in ("dojo_num_state", "dojo_num_input", "dojo_num_residual", "dojo_num_grad_state", "dojo_shared_bytes_per_env"):
        getattr(L, n).argtypes = [vp]
        getattr(L, n).restype = C.c_int
    L.dojo_launch_count.argtypes = [vp]
    L.dojo_launch_count.restype = C.c_int64
    L.dojo_step.argtypes = [vp, op, C.c_int, vp, vp, vp, vp, vp, vp, vp, C.c_uint32]
    L.dojo_step.restype = C.c_int
    L.dojo_step_async.argtypes = [vp, op, C.c_int, vp, vp, vp, vp, vp, vp, vp, C.c_uint32, vp]
    L.dojo_step_async.restype = C.c_int
    L.dojo_step_trace.argtypes = [vp, op, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, C.c_uint32]
    L.dojo_step_trace.restype = C.c_int
    L.dojo_step_trace_async.argtypes = [vp, op, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, C.c_uint32, vp]
    L.dojo_step_trace_async.restype = C.c_int
    L.dojo_step_grad.argtypes = [vp, op, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, C.c_uint32]
    L.dojo_step_grad.restype = C.c_int
    L.dojo_step_grad_async.argtypes = [vp, op, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, C.c_uint32, vp]
    L.dojo_step_grad_async.restype = C.c_int
    L.dojo_rollout.argtypes = [vp, op, C.c_int, C.c_int, vp, vp, vp, vp, vp]
    L.dojo_rollout.restype = C.c_int
    L.dojo_rollout_async.argtypes = [vp, op, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp]
    L.dojo_rollout_async.restype = C.c_int
    L.dojo_num_minimal.argtypes = [vp]
    L.dojo_num_minimal.restype = C.c_int
    for name in ("dojo_minimal_to_maximal", "dojo_maximal_to_minimal"):
        getattr(L, name).argtypes = [vp, C.c_int, vp, vp]
        getattr(L, name).restype = C.c_int
        getattr(L, name + "_async").argtypes = [vp, C.c_int, vp, vp, vp]
        getattr(L, name + "_async").restype = C.c_int
    L.dojo_step_minimal.argtypes = [vp, op, C.c_int, vp, vp, vp, vp, vp]
    L.dojo_step_minimal.restype = C.c_int
    L.dojo_step_minimal_flags.argtypes = [vp, op, C.c_int, vp, vp, vp, vp, vp, C.c_uint32]
    L.dojo_step_minimal_flags.restype = C.c_int
    for name in ("dojo_maximal_to_minimal_jacobian", "dojo_minimal_to_maximal_jacobian"):
        getattr(L, name).argtypes = [vp, C.c_int, vp, vp]
        getattr(L, name).restype = C.c_int
        getattr(L, name + "_async").argtypes = [vp, C.c_int, vp, vp, vp]
        getattr(L, name + "_async").restype = C.c_int
    L.dojo_minimal_gradients.argtypes = [vp, op, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    L.dojo_minimal_gradients.restype = C.c_int
    ep = C.POINTER(capi.DojoEnvSpec)
    for name in ("dojo_env_num_state", "dojo_env_num_action"):
        getattr(L, name).argtypes = [vp, ep]
        getattr(L, name).restype = C.c_int
    L.dojo_env_step.argtypes = [vp, op, ep, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    L.dojo_env_step.restype = C.c_int
    L.dojo_env_step_async.argtypes = [vp, op, ep, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.dojo_env_step_async.restype = C.c_int
    L.dojo_env_reset.argtypes = [vp, ep, C.c_int, vp, vp, vp]
    L.dojo_env_reset.restype = C.c_int
    L.dojo_env_rollout.argtypes = [vp, op, ep, C.c_int, C.c_int, vp, vp, vp, vp, vp]
    L.dojo_env_rollout.restype = C.c_int
    L.dojo_env_policy_rollout.argtypes = [vp, op, ep, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.dojo_env_policy_rollout.restype = C.c_int
    L.dojo_num_contact_data.argtypes = [vp]
    L.dojo_num_contact_data.restype = C.c_int
    L.dojo_step_grad_contact.argtypes = [vp, op, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.dojo_step_grad_contact.restype = C.c_int
    L.dojo_step_grad_contact_async.argtypes = [vp, op, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_uint32, vp]
    L.dojo_step_grad_contact_async.restype = C.c_int
    L.dojo_update_params.argtypes = [vp, C.POINTER(capi.DojoMechanismDesc)]
    L.dojo_update_params.restype = C.c_int
    L.dojo_step_record.argtypes = [vp, op, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    L.dojo_step_record.restype = C.c_int
    L.dojo_step_record_async.argtypes = [vp, op, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.dojo_step_record_async.restype = C.c_int
    L.dojo_simulate_record.argtypes = [vp, op, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    L.dojo_simulate_record.restype = C.c_int
    L.dojo_rollout_grad.argtypes = [vp, op, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    L.dojo_rollout_grad.restype = C.c_int
    L.dojo_rollout_grad_async.argtypes = [vp, op, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.dojo_rollout_grad_async.restype = C.c_int
    L.dojo_rollout_minimal_gradients.argtypes = [vp, op, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    L.dojo_rollout_minimal_gradients.restype = C.c_int
    fp = C.POINTER(capi.DojoFeedback)
    L.dojo_rollout_feedback.argtypes = [vp, op, C.c_int, C.c_int, vp, fp, vp, vp, vp, vp, vp]
    L.dojo_rollout_feedback.restype = C.c_int
    L.dojo_rollout_feedback_async.argtypes = [vp, op, C.c_int, C.c_int, vp, fp, vp, vp, vp, vp, vp, vp]
    L.dojo_rollout_feedback_async.restype = C.c_int
    cp = C.POINTER(capi.DojoQuadraticCost)
    L.dojo_lqr_backward.argtypes = [vp, C.c_int, C.c_int, cp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.dojo_lqr_backward.restype = C.c_int
    L.dojo_lqr_backward_async.argtypes = [vp, C.c_int, C.c_int, cp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.dojo_lqr_backward_async.restype = C.c_int
    L.dojo_gather_create.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
    L.dojo_gather_create.restype = C.c_int
    L.dojo_gather_export.argtypes = [vp, vp]
    L.dojo_gather_export.restype = C.c_int
    L.dojo_gather_connect.argtypes = [vp, vp]
    L.dojo_gather_connect.restype = C.c_int
    L.dojo_gather_buffer.argtypes = [vp]
    L.dojo_gather_buffer.restype = vp
    L.dojo_gather_destroy.argtypes = [vp]
    L.dojo_gather_destroy.restype = C.c_int
    L.dojo_step_gather_async.argtypes = [vp, vp, op, C.c_int, vp, vp, vp, vp, vp, vp, C.c_uint32, vp]
    L.dojo_step_gather_async.restype = C.c_int
    L.dojo_step_grad_gather_async.argtypes = [vp, vp, op, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, C.c_uint32, vp]
    L.dojo_step_grad_gather_async.restype = C.c_int
    _lib = L
    return L


def _p(a):
    """numpy array / int (device pointer) / None -> c_void_p"""
    if a is None:
        return None
    if isinstance(a, (int, np.integer)):
        return C.c_void_p(int(a))
    return C.c_void_p(a.ctypes.data)


def _entries(T: int, B: int, arrays: dict, what: str):
    """Broadcast {name: (array or None, tail shape)} to one (steps, envs): each array is given as tail, (B,) + tail or (T, 1 or B) + tail
    and is broadcast to the largest given.  Returns (steps, envs, {name: C-contiguous [steps, envs] + tail, matrices column-major per
    entry}) for the given arrays."""
    def lead(a, tail):
        a = np.asarray(a, dtype=np.float64)
        n = a.ndim - len(tail)
        if a.shape[n:] != tail or n < 0 or n > 2 or (n == 1 and a.shape[0] != B) or (n == 2 and (a.shape[0] != T or a.shape[1] not in (1, B))):
            raise ValueError(f"{what} array of shape {a.shape}: expected {tail}, (B,) + {tail} or (T, 1 or B) + {tail} with T = {T}, B = {B}")
        return a.reshape(((1, 1), (1, B), a.shape[:2])[n] + tail)
    given = {k: (lead(v, tail), tail) for k, (v, tail) in arrays.items() if v is not None}
    steps = max(a.shape[0] for a, _ in given.values())
    envs = max(a.shape[1] for a, _ in given.values())
    out = {}
    for k, (a, tail) in given.items():
        a = np.broadcast_to(a, (steps, envs) + tail)
        out[k] = np.ascontiguousarray(a.swapaxes(2, 3) if a.ndim == 4 else a)
    return steps, envs, out


def feedback_arrays(T: int, B: int, nu: int, K, x_ref=None, u_ref=None, K_i=None):
    """The arrays of a DojoFeedback from the shapes BatchedStepper.rollout_feedback accepts: a matrix (K, K_i) as [nu, 2nu], [B, nu, 2nu],
    [T, 1, nu, 2nu] or [T, B, nu, 2nu], a vector (x_ref [2nu], u_ref [nu]) likewise.  All arrays share one (steps, envs): each is broadcast
    to the largest given.  Returns (steps, envs, K, x_ref, u_ref, K_i) with every given array C-contiguous [steps, envs, ...] and the
    matrices column-major per entry ([steps, envs, 2nu, nu]); absent arrays stay None."""
    steps, envs, out = _entries(T, B, {"K": (K, (nu, 2 * nu)), "x_ref": (x_ref, (2 * nu,)), "u_ref": (u_ref, (nu,)), "K_i": (K_i, (nu, 2 * nu))},
                                "feedback")
    return steps, envs, out["K"], out.get("x_ref"), out.get("u_ref"), out.get("K_i")


def cost_arrays(T: int, B: int, nu: int, Q, R, x_goal=None, u_goal=None, Q_final=None, x_goal_final=None):
    """The arrays of a DojoQuadraticCost, with the broadcasting rules of feedback_arrays: Q [2nu, 2nu], R [nu, nu], x_goal [2nu] and
    u_goal [nu], each also per environment ([B, ...]) or per step ([T, 1 or B, ...]), broadcast to one (steps, envs); Q_final [2nu, 2nu]
    and x_goal_final [2nu], each also [B, ...], broadcast to envs.  Q_final defaults to the last step's Q and x_goal_final to the last
    step's x_goal.  Returns (steps, envs, Q, R, x_goal, u_goal, Q_final, x_goal_final), C-contiguous, Q / R as [steps, envs, n, n] and
    Q_final as [envs, 2nu, 2nu] column-major per entry (Q, R, Q_final symmetric in use); absent goals stay None."""
    nx = 2 * nu
    steps, envs, out = _entries(T, B, {"Q": (Q, (nx, nx)), "R": (R, (nu, nu)), "x_goal": (x_goal, (nx,)), "u_goal": (u_goal, (nu,))}, "cost")
    fin = {}
    for k, a, tail in (("Q_final", Q_final, (nx, nx)), ("x_goal_final", x_goal_final, (nx,))):
        if a is not None:
            a = np.asarray(a, dtype=np.float64)
            if a.shape not in (tail, (B,) + tail):
                raise ValueError(f"final cost array of shape {a.shape}: expected {tail} or (B,) + {tail} with B = {B}")
            fin[k] = a.reshape((1,) + tail if a.ndim == len(tail) else a.shape)
    if any(a.shape[0] > envs for a in fin.values()):  # a per-environment final cost makes the running cost per environment too
        envs = B
        out = {k: np.ascontiguousarray(np.broadcast_to(a, (steps, envs) + a.shape[2:])) for k, a in out.items()}
    for k, a in fin.items():
        a = np.broadcast_to(a, (envs,) + a.shape[1:])
        fin[k] = np.ascontiguousarray(a.swapaxes(1, 2) if a.ndim == 3 else a)
    Qf = fin.get("Q_final", out["Q"][-1])
    xgf = fin.get("x_goal_final", None if x_goal is None else out["x_goal"][-1])
    return steps, envs, out["Q"], out["R"], out.get("x_goal"), out.get("u_goal"), Qf, xgf


class BatchedStepper:
    """A mechanism bound to one GPU: the handle of include/dojo_b200.h.

    Host arrays are [B, feature] C-contiguous numpy arrays, i.e. exactly the column-major
    [feature x B] Julia matrices of the ABI.  Device buffers are passed as integer pointers
    (``tensor.data_ptr()``) to the *_device methods together with a CUDA stream handle.
    """

    def __init__(self, mech: Mechanism, max_batch: int, device: int = 0):
        self.mech = mech
        self.L = load_library()
        desc, keep = capi.flatten(mech)
        h = C.c_void_p()
        rc = self.L.dojo_create(C.byref(desc), int(device), int(max_batch), C.byref(h))
        if rc != 0:
            msg = self.L.dojo_last_error(None).decode()
            raise RuntimeError(f"dojo_create failed ({rc}): {msg}")
        self.h = h
        self.max_batch = int(max_batch)
        self.device = int(device)
        self.nz = self.L.dojo_num_state(h)
        self.nu = self.L.dojo_num_input(h)
        self.nres = self.L.dojo_num_residual(h)
        self.ngrad = self.L.dojo_num_grad_state(h)
        assert (self.nz, self.nu, self.nres) == (mech.nz, mech.nu, mech.nres)

    def close(self):
        if getattr(self, "h", None):
            self.L.dojo_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            raise RuntimeError(f"{what} failed ({rc}): {self.L.dojo_last_error(self.h).decode()}")

    def update_params(self, mech: Mechanism):
        """Swap in the parameters of `mech` (same topology: bodies, joints, joint types, limits, contacts) without re-creating
        the handle -- the system-identification loop of examples/system_identification/utilities.jl:41-87."""
        desc, keep = capi.flatten(mech)
        self._check(self.L.dojo_update_params(self.h, C.byref(desc)), "dojo_update_params")
        self.mech = mech

    @property
    def shared_bytes_per_env(self) -> int:
        return self.L.dojo_shared_bytes_per_env(self.h)

    @property
    def launch_config(self) -> dict:
        """Launch configuration chosen by dojo_create (diagnostics; dojo_debug_config is not part of the public header)."""
        out = (C.c_int * 17)()
        self.L.dojo_debug_config.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
        self.L.dojo_debug_config(self.h, out)
        keys = ("slots", "slots_grad", "grad_chunk", "arena_bytes", "grad_arena_bytes", "smem_fwd", "smem_grad", "plan_smem_mask", "plan_smem_mask_grad",
                "ls_pair", "phases", "steps", "plan_blob_bytes", "warps_per_env", "ctas_per_sm", "ctas_per_sm_grad", "small_step")
        return dict(zip(keys, list(out)))

    @property
    def launch_count(self) -> int:
        return int(self.L.dojo_launch_count(self.h))

    # ------------------------------------------------------------------ host buffers
    def step(self, Z, U=None, opts: Optional[capi.DojoSolverOptions] = None, fext=None, flags: int = 0, return_sol: bool = False, out=None,
             trace: bool = False):
        """One step! of every environment.  Host arrays in, host arrays out; page-locked arrays (e.g. views of torch pinned
        tensors) are copied from / to directly, pageable ones go through the library's pinned staging buffers.
        out = (Z_next, status, iters) reuses caller-provided result arrays.
        trace=True runs the traced step (dojo_step_trace, same results) and appends trace [B, max_iter, 5] to the returned tuple:
        one row per loop head of the solver, (rvio, bvio, alpha, mu, trials), NaN after the last head reached (include/dojo_b200.h)."""
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=np.float64)
        B = Z.shape[0]
        assert Z.shape[1] == self.nz
        U = np.zeros((B, self.nu)) if U is None else np.ascontiguousarray(np.atleast_2d(U), dtype=np.float64)
        assert U.shape == (B, self.nu)
        if fext is not None:
            fext = np.ascontiguousarray(fext, dtype=np.float64).reshape(B, 6 * self.mech.Nb)
        if out is not None:
            Zn, status, iters = out
            assert Zn.shape == Z.shape and Zn.dtype == np.float64 and Zn.flags.c_contiguous
            assert status.shape == (B,) and status.dtype == np.int32 and iters.shape == (B,) and iters.dtype == np.int32
        else:
            Zn = np.empty_like(Z)
            status = np.zeros(B, dtype=np.int32)
            iters = np.zeros(B, dtype=np.int32)
        sol = np.empty((B, self.nres)) if return_sol else None
        o = opts if opts is not None else capi.solver_options()
        if trace:
            tr = np.empty((B, max(int(o.max_iter), 0), 5))
            rc = self.L.dojo_step_trace(self.h, C.byref(o), B, _p(Z), _p(U), _p(fext), _p(Zn), _p(sol), _p(status), _p(iters), _p(tr), flags)
            self._check(rc, "dojo_step_trace")
            return (Zn, status, iters, sol, tr) if return_sol else (Zn, status, iters, tr)
        rc = self.L.dojo_step(self.h, C.byref(o), B, _p(Z), _p(U), _p(fext), _p(Zn), _p(sol), _p(status), _p(iters), flags)
        self._check(rc, "dojo_step")
        return (Zn, status, iters, sol) if return_sol else (Zn, status, iters)

    def step_grad(self, Z, U=None, opts=None, flags: int = 0, out=None):
        """step! + IFT gradients.  Returns (Z_next, Fz [B, 12Nb, 12Nb], Fu [B, 12Nb, nu], status, iters) with Fz[e] = dz'/dz.
        out = (Z_next, Fz_raw [B, 12Nb, 12Nb], Fu_raw [B, nu, 12Nb], status, iters) reuses caller buffers (e.g. page-locked
        ones); the raw arrays hold each environment's Jacobian column-major, the returned Fz / Fu are transposed views."""
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=np.float64)
        B = Z.shape[0]
        U = np.zeros((B, self.nu)) if U is None else np.ascontiguousarray(np.atleast_2d(U), dtype=np.float64)
        ng = self.ngrad
        if out is not None:
            Zn, Fz, Fu, status, iters = out
            assert Zn.shape == Z.shape and Fz.shape == (B, ng, ng) and Fu.shape == (B, self.nu, ng)
            assert all(a.flags.c_contiguous for a in (Zn, Fz, Fu, status, iters)) and status.dtype == np.int32 and iters.dtype == np.int32
        else:
            Zn = np.empty_like(Z)
            Fz = np.empty((B, ng, ng))   # per env column-major [ng x ng]  ==  Fz[e].T is the Jacobian
            Fu = np.empty((B, self.nu, ng))
            status = np.zeros(B, dtype=np.int32)
            iters = np.zeros(B, dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_step_grad(self.h, C.byref(o), B, _p(Z), _p(U), None, _p(Zn), _p(Fz), _p(Fu), _p(status), _p(iters), flags)
        self._check(rc, "dojo_step_grad")
        return Zn, np.transpose(Fz, (0, 2, 1)), np.transpose(Fu, (0, 2, 1)), status, iters

    def step_grad_contact(self, Z, U=None, opts=None):
        """step! + get_contact_gradients (gradients/contact.jl:1-55).  Returns (Z_next, Fz [B, 12Nb, 12Nb], Fu [B, 12Nb, nu],
        Fc [B, 12Nb, 5Ni] = dz'/d[friction_coefficient, contact_radius, contact_origin(3)] per contact, status, iters)."""
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=np.float64)
        B = Z.shape[0]
        U = np.zeros((B, self.nu)) if U is None else np.ascontiguousarray(np.atleast_2d(U), dtype=np.float64)
        ng, nc = self.ngrad, self.L.dojo_num_contact_data(self.h)
        Zn = np.empty_like(Z)
        Fz, Fu, Fc = np.empty((B, ng, ng)), np.empty((B, self.nu, ng)), np.empty((B, nc, ng))
        status, iters = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_step_grad_contact(self.h, C.byref(o), B, _p(Z), _p(U), _p(Zn), _p(Fz), _p(Fu), _p(Fc), _p(status), _p(iters))
        self._check(rc, "dojo_step_grad_contact")
        return Zn, np.transpose(Fz, (0, 2, 1)), np.transpose(Fu, (0, 2, 1)), np.transpose(Fc, (0, 2, 1)), status, iters

    def rollout(self, Z0, U=None, T: int = 1, opts=None, record: bool = False):
        Z0 = np.ascontiguousarray(np.atleast_2d(Z0), dtype=np.float64)
        B = Z0.shape[0]
        if U is not None:
            U = np.ascontiguousarray(U, dtype=np.float64)
            assert U.shape == (T, B, self.nu)
        Zf = np.empty_like(Z0)
        traj = np.empty((T, B, self.nz)) if record else None
        st = np.zeros(B, dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_rollout(self.h, C.byref(o), B, int(T), _p(Z0), _p(U), _p(Zf), _p(traj), _p(st))
        self._check(rc, "dojo_rollout")
        return (Zf, st, traj) if record else (Zf, st)

    def rollout_grad(self, Z0, U=None, T: int = 1, opts=None):
        """T fused steps and the IFT Jacobians of every step (dojo_rollout_grad): simulate! + get_maximal_gradients! at each step.
        U [T, B, nu] or None.  Returns (Z_traj [T+1, B, 13Nb] with Z_traj[0] = Z0 and Z_traj[t+1] the state after step t,
        Fz [T, B, 12Nb, 12Nb], Fu [T, B, 12Nb, nu] with Fz[t, e] = dz_{t+1}/dz_t, status [T, B], iters [T, B]); Fz / Fu are transposed
        views of the column-major per-pair buffers, as in step_grad."""
        Z0 = np.ascontiguousarray(np.atleast_2d(Z0), dtype=np.float64)
        B, T, ng = Z0.shape[0], int(T), self.ngrad
        assert Z0.shape[1] == self.nz
        if U is not None:
            U = np.ascontiguousarray(U, dtype=np.float64)
            assert U.shape == (T, B, self.nu)
        traj = np.empty((max(T, 0) + 1, B, self.nz))
        Fz, Fu = np.empty((max(T, 0), B, ng, ng)), np.empty((max(T, 0), B, self.nu, ng))
        status, iters = np.zeros((max(T, 0), B), dtype=np.int32), np.zeros((max(T, 0), B), dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_rollout_grad(self.h, C.byref(o), B, T, _p(Z0), _p(U), _p(traj), _p(Fz), _p(Fu), _p(status), _p(iters))
        self._check(rc, "dojo_rollout_grad")
        return traj, np.transpose(Fz, (0, 1, 3, 2)), np.transpose(Fu, (0, 1, 3, 2)), status, iters

    def rollout_minimal_gradients(self, X0, U=None, T: int = 1, opts=None):
        """The same in minimal coordinates (dojo_rollout_minimal_gradients): the rollout from minimal_to_maximal(X0) and
        get_minimal_gradients! at every step.  Returns (X_traj [T+1, B, 2nu], Gx [T, B, 2nu, 2nu], Gu [T, B, 2nu, nu], status [T, B],
        iters [T, B])."""
        X0 = np.ascontiguousarray(np.atleast_2d(X0), dtype=np.float64)
        B, T, nm = X0.shape[0], int(T), self.nmin
        assert X0.shape[1] == nm
        if U is not None:
            U = np.ascontiguousarray(U, dtype=np.float64)
            assert U.shape == (T, B, self.nu)
        Xt = np.empty((max(T, 0) + 1, B, nm))
        Gx, Gu = np.empty((max(T, 0), B, nm, nm)), np.empty((max(T, 0), B, self.nu, nm))
        status, iters = np.zeros((max(T, 0), B), dtype=np.int32), np.zeros((max(T, 0), B), dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_rollout_minimal_gradients(self.h, C.byref(o), B, T, _p(X0), _p(U), _p(Xt), _p(Gx), _p(Gu), _p(status), _p(iters))
        self._check(rc, "dojo_rollout_minimal_gradients")
        return Xt, np.transpose(Gx, (0, 1, 3, 2)), np.transpose(Gu, (0, 1, 3, 2)), status, iters

    def rollout_feedback(self, Z0, T: int, K, x_ref=None, u_ref=None, K_i=None, xi=None, opts=None, record: bool = False):
        """Closed-loop rollout (dojo_rollout_feedback): before every step t the device maps the state to minimal coordinates x_t and applies
        u_t = u_ref - K (x_t - x_ref) - K_i xi_t with xi_t = xi_{t-1} + h (x_t - x_ref), in the one launch of dojo_rollout.  K / K_i as
        [nu, 2nu], [B, nu, 2nu], [T, 1, nu, 2nu] or [T, B, nu, 2nu], x_ref / u_ref likewise (feedback_arrays); xi [B, 2nu] or [2nu]
        (zero when K_i is given without it).  Returns (Z_final [B, 13Nb], status_any [B], Z_traj [T, B, 13Nb] or None (record=False),
        U_applied [T, B, nu], xi [B, 2nu] or None (no K_i)).  dojo_rollout(Z0, U_applied) reproduces the trajectory bit for bit."""
        Z0 = np.ascontiguousarray(np.atleast_2d(Z0), dtype=np.float64)
        B, T = Z0.shape[0], int(T)
        assert Z0.shape[1] == self.nz
        steps, envs, Kc, xr, ur, Kic = feedback_arrays(T, B, self.nu, K, x_ref, u_ref, K_i)
        fb = capi.DojoFeedback(steps, envs, capi.dptr(Kc), None if Kic is None else capi.dptr(Kic), None if xr is None else capi.dptr(xr),
                               None if ur is None else capi.dptr(ur))
        if Kic is not None:
            xi = np.zeros((B, 2 * self.nu)) if xi is None else np.array(np.broadcast_to(np.asarray(xi, dtype=np.float64), (B, 2 * self.nu)))
        else:
            xi = None
        Zf = np.empty_like(Z0)
        traj = np.empty((T, B, self.nz)) if record and T > 0 else None
        Ua = np.empty((max(T, 0), B, self.nu))
        st = np.zeros(B, dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_rollout_feedback(self.h, C.byref(o), B, T, _p(Z0), C.byref(fb), _p(xi), _p(Zf), _p(traj), _p(Ua), _p(st))
        self._check(rc, "dojo_rollout_feedback")
        return Zf, st, traj, Ua, xi

    def lqr_backward(self, X_traj, U, Gx, Gu, cost, mu=None, active=None):
        """Riccati backward pass of iLQR / TVLQR (dojo_lqr_backward) on the shapes rollout_minimal_gradients returns: X_traj [T+1, B, 2nu],
        U [T, B, nu] or None, Gx [T, B, 2nu, 2nu], Gu [T, B, 2nu, nu].  cost has the attributes Q, R, x_goal, u_goal, Q_final,
        x_goal_final (api.QuadraticCost; shapes as cost_arrays).  mu [B] or a scalar (None: 0); active [nu] mask (None: all inputs).
        Returns (K [T, B, nu, 2nu], k [T, B, nu], dV [B, 2], status [B]): the law u = u_bar + alpha k - K (x - x_bar), the expected
        decrease alpha dV[0] + alpha^2 dV[1], and per environment 0 or t + 1 when the Cholesky of Quu + mu I failed at step t (then its
        K[:t+1], k[:t+1] and dV are NaN)."""
        X_traj = np.ascontiguousarray(X_traj, dtype=np.float64)
        T, B, nx = X_traj.shape[0] - 1, X_traj.shape[1], 2 * self.nu
        assert X_traj.shape[2] == nx and T >= 1
        Gx, Gu = np.asarray(Gx, dtype=np.float64), np.asarray(Gu, dtype=np.float64)
        assert Gx.shape == (T, B, nx, nx) and Gu.shape == (T, B, nx, self.nu)
        Gxc, Guc = np.ascontiguousarray(Gx.swapaxes(2, 3)), np.ascontiguousarray(Gu.swapaxes(2, 3))  # column-major per pair
        if U is not None:
            U = np.ascontiguousarray(U, dtype=np.float64)
            assert U.shape == (T, B, self.nu)
        ca = cost_arrays(T, B, self.nu, cost.Q, cost.R, cost.x_goal, cost.u_goal, cost.Q_final, cost.x_goal_final)
        c = capi.quadratic_cost(*ca)
        mu = None if mu is None else np.ascontiguousarray(np.broadcast_to(np.asarray(mu, dtype=np.float64), (B,)))
        act = None if active is None else np.ascontiguousarray(np.asarray(active).astype(np.int32).reshape(self.nu))
        K, k, dV, st = np.empty((T, B, nx, self.nu)), np.empty((T, B, self.nu)), np.empty((B, 2)), np.zeros(B, dtype=np.int32)
        rc = self.L.dojo_lqr_backward(self.h, B, T, C.byref(c), _p(act), _p(X_traj), _p(U), _p(Gxc), _p(Guc), _p(mu), _p(K), _p(k), _p(dV), _p(st))
        self._check(rc, "dojo_lqr_backward")
        return np.transpose(K, (0, 1, 3, 2)), k, dV, st

    # ------------------------------------------------------------------ minimal coordinates (SURVEY 8 f1)
    @property
    def nmin(self) -> int:
        return self.L.dojo_num_minimal(self.h)

    def minimal_to_maximal(self, X):
        """minimal_to_maximal (mechanism/state.jl:9-22), batched: X [B, 2 nu] -> Z [B, 13 Nb]."""
        X = np.ascontiguousarray(np.atleast_2d(X), dtype=np.float64)
        assert X.shape[1] == self.nmin
        Z = np.empty((X.shape[0], self.nz))
        self._check(self.L.dojo_minimal_to_maximal(self.h, X.shape[0], _p(X), _p(Z)), "dojo_minimal_to_maximal")
        return Z

    def maximal_to_minimal(self, Z):
        """maximal_to_minimal (mechanism/state.jl:44-66), batched: Z [B, 13 Nb] -> X [B, 2 nu]."""
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=np.float64)
        assert Z.shape[1] == self.nz
        X = np.empty((Z.shape[0], self.nmin))
        self._check(self.L.dojo_maximal_to_minimal(self.h, Z.shape[0], _p(Z), _p(X)), "dojo_maximal_to_minimal")
        return X

    def step_minimal(self, X, U=None, opts=None, flags: int = 0):
        """step_minimal_coordinates! (simulation/step.jl:42-61), batched.  Returns (X_next, status, iters).  flags =
        DOJO_FLAG_Q1_LITERAL_RETURN: the reference's literal return value (SURVEY.md Q1) in minimal coordinates."""
        X = np.ascontiguousarray(np.atleast_2d(X), dtype=np.float64)
        B = X.shape[0]
        U = None if U is None else np.ascontiguousarray(np.atleast_2d(U), dtype=np.float64)
        Xn = np.empty_like(X)
        status, iters = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        self._check(self.L.dojo_step_minimal_flags(self.h, C.byref(o), B, _p(X), _p(U), _p(Xn), _p(status), _p(iters), C.c_uint32(flags)), "dojo_step_minimal")
        return Xn, status, iters

    def maximal_to_minimal_jacobian(self, Z):
        """maximal_to_minimal_jacobian (gradients/state.jl:9-56), batched: Z [B, 13 Nb] -> M [B, 2 nu, 12 Nb]."""
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=np.float64)
        assert Z.shape[1] == self.nz
        J = np.empty((Z.shape[0], self.ngrad, self.nmin))  # column-major [2 nu x 12 Nb] per environment
        self._check(self.L.dojo_maximal_to_minimal_jacobian(self.h, Z.shape[0], _p(Z), _p(J)), "dojo_maximal_to_minimal_jacobian")
        return np.transpose(J, (0, 2, 1))

    def minimal_to_maximal_jacobian(self, Z):
        """minimal_to_maximal_jacobian (gradients/state.jl:136-179) evaluated at the maximal states Z [B, 13 Nb]
        (= minimal_to_maximal(X)): N [B, 12 Nb, 2 nu]."""
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=np.float64)
        assert Z.shape[1] == self.nz
        J = np.empty((Z.shape[0], self.nmin, self.ngrad))  # column-major [12 Nb x 2 nu] per environment
        self._check(self.L.dojo_minimal_to_maximal_jacobian(self.h, Z.shape[0], _p(Z), _p(J)), "dojo_minimal_to_maximal_jacobian")
        return np.transpose(J, (0, 2, 1))

    def minimal_gradients(self, X, U=None, opts=None):
        """get_minimal_gradients! (gradients/state.jl:182-217), batched.
        Returns (X_next [B, 2nu], dx'/dx [B, 2nu, 2nu], dx'/du [B, 2nu, nu], status, iters)."""
        X = np.ascontiguousarray(np.atleast_2d(X), dtype=np.float64)
        B = X.shape[0]
        assert X.shape[1] == self.nmin
        U = None if U is None else np.ascontiguousarray(np.atleast_2d(U), dtype=np.float64)
        Xn = np.empty_like(X)
        Gx = np.empty((B, self.nmin, self.nmin))
        Gu = np.empty((B, self.nu, self.nmin))
        status, iters = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_minimal_gradients(self.h, C.byref(o), B, _p(X), _p(U), _p(Xn), _p(Gx), _p(Gu), _p(status), _p(iters))
        self._check(rc, "dojo_minimal_gradients")
        return Xn, np.transpose(Gx, (0, 2, 1)), np.transpose(Gu, (0, 2, 1)), status, iters

    # ------------------------------------------------------------------ trajectory recording / diagnostics (SURVEY 8 f3)
    def step_record(self, Z, U=None, opts=None):
        """step! + save_to_storage! (simulation/storage.jl:50-67).  Returns (Z_next, storage [B, Nb, 12] = px pq vl wl per body,
        diag [B, 8] = linear momentum, angular momentum about the centre of mass, kinetic, potential energy, status, iters)."""
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=np.float64)
        B = Z.shape[0]
        U = None if U is None else np.ascontiguousarray(np.atleast_2d(U), dtype=np.float64)
        Zn = np.empty_like(Z)
        sto, diag = np.empty((B, self.mech.Nb, 12)), np.empty((B, 8))
        status, iters = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_step_record(self.h, C.byref(o), B, _p(Z), _p(U), _p(Zn), _p(sto), _p(diag), _p(status), _p(iters))
        self._check(rc, "dojo_step_record")
        return Zn, sto, diag, status, iters

    def simulate_record(self, Z0, U=None, T: int = 1, opts=None):
        """simulate!(...; record=true) with open-loop inputs U [T, B, nu].  Returns (Z_final, Z_traj [T, B, 13Nb] = the state
        before every solve (Storage.x, q, v, w), storage [T, B, Nb, 12], diag [T, B, 8], status_any)."""
        Z0 = np.ascontiguousarray(np.atleast_2d(Z0), dtype=np.float64)
        B = Z0.shape[0]
        if U is not None:
            U = np.ascontiguousarray(U, dtype=np.float64)
            assert U.shape == (T, B, self.nu)
        Zf = np.empty_like(Z0)
        traj, sto, diag = np.empty((T, B, self.nz)), np.empty((T, B, self.mech.Nb, 12)), np.empty((T, B, 8))
        st = np.zeros(B, dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_simulate_record(self.h, C.byref(o), B, int(T), _p(Z0), _p(U), _p(Zf), _p(traj), _p(sto), _p(diag), _p(st))
        self._check(rc, "dojo_simulate_record")
        return Zf, traj, sto, diag, st

    def step_record_device(self, dZ: int, dU: Optional[int], dZn: int, dstorage: int, ddiag: int, B: int, opts=None, dstatus=None, diters=None, stream: int = 0):
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_step_record_async(self.h, C.byref(o), int(B), _p(dZ), _p(dU), _p(dZn), _p(dstorage), _p(ddiag), _p(dstatus), _p(diters),
                                           C.c_void_p(int(stream)))
        self._check(rc, "dojo_step_record_async")

    # ------------------------------------------------------------------ environment layer (SURVEY 8 f2)
    def env_sizes(self, spec):
        return self.L.dojo_env_num_state(self.h, C.byref(spec)), self.L.dojo_env_num_action(self.h, C.byref(spec))

    def env_step(self, spec, S, A=None, opts=None):
        """step!(environment, s, a) + get_state + reward + failure test for a batch (DojoEnvironments/src/environments.jl:77-109,
        examples/learning/ant_ars.jl:79-116).  S [B, ns], A [B, na] -> (S_next, reward, done, status, iters)."""
        ns, na = self.env_sizes(spec)
        S = np.ascontiguousarray(np.atleast_2d(S), dtype=np.float64)
        B = S.shape[0]
        assert S.shape[1] == ns
        if A is not None:
            A = np.ascontiguousarray(np.atleast_2d(A), dtype=np.float64)
            assert A.shape == (B, na)
        Sn = np.empty_like(S)
        reward = np.empty(B)
        done, status, iters = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_env_step(self.h, C.byref(o), C.byref(spec), B, _p(S), _p(A), _p(Sn), _p(reward), _p(done), _p(status), _p(iters))
        self._check(rc, "dojo_env_step")
        return Sn, reward, done, status, iters

    def env_step_device(self, spec, dS: int, dA: Optional[int], dSn: int, B: int, opts=None, dreward=None, ddone=None, dstatus=None, diters=None,
                        stream: int = 0):
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_env_step_async(self.h, C.byref(o), C.byref(spec), int(B), _p(dS), _p(dA), _p(dSn), _p(dreward), _p(ddone), _p(dstatus),
                                        _p(diters), C.c_void_p(int(stream)))
        self._check(rc, "dojo_env_step_async")

    def env_rollout(self, spec, S0, A=None, T: int = 1, opts=None):
        """Open-loop rollout of T environment steps on the device (examples/learning/ant_ars.jl:79-116 without the policy):
        S0 [B, ns], A [T, B, na] -> (S_final, return [B], failed [B])."""
        ns, na = self.env_sizes(spec)
        S0 = np.ascontiguousarray(np.atleast_2d(S0), dtype=np.float64)
        B = S0.shape[0]
        if A is not None:
            A = np.ascontiguousarray(A, dtype=np.float64)
            assert A.shape == (T, B, na)
        Sf, ret, failed = np.empty_like(S0), np.empty(B), np.zeros(B, dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_env_rollout(self.h, C.byref(o), C.byref(spec), B, int(T), _p(S0), _p(A), _p(Sf), _p(ret), _p(failed))
        self._check(rc, "dojo_env_rollout")
        return Sf, ret, failed

    def env_policy_rollout(self, spec, S0, Theta, T: int, mean=None, std=None, opts=None, record_states: bool = False):
        """Closed-loop rollout with one linear policy per environment (ARS evaluation): Theta [B, na, ns], a = Theta_e ((s - mean) / std).
        Returns (S_final, return [B], failed [B]) and, with record_states, the states observed before every step [T, B, ns]."""
        ns, na = self.env_sizes(spec)
        S0 = np.ascontiguousarray(np.atleast_2d(S0), dtype=np.float64)
        B = S0.shape[0]
        Theta = np.asarray(Theta, dtype=np.float64)
        assert Theta.shape == (B, na, ns)
        ThetaC = np.ascontiguousarray(Theta.transpose(0, 2, 1))  # column-major [na x ns] per environment
        mean = None if mean is None else np.ascontiguousarray(mean, dtype=np.float64)
        std = None if std is None else np.ascontiguousarray(std, dtype=np.float64)
        Sf, ret, failed = np.empty_like(S0), np.empty(B), np.zeros(B, dtype=np.int32)
        traj = np.empty((T, B, ns)) if record_states else None
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_env_policy_rollout(self.h, C.byref(o), C.byref(spec), B, int(T), _p(S0), _p(ThetaC), _p(mean), _p(std), _p(Sf), _p(ret),
                                            _p(failed), _p(traj))
        self._check(rc, "dojo_env_policy_rollout")
        return (Sf, ret, failed, traj) if record_states else (Sf, ret, failed)

    def env_reset(self, spec, S, s0, mask=None):
        """S[e] = s0 where mask[e] != 0 (all if mask is None).  S / mask: numpy arrays (in place) or device pointers + B."""
        s0 = np.ascontiguousarray(s0, dtype=np.float64)
        if isinstance(S, tuple):  # (device pointer, B)
            dS, B = S
            self._check(self.L.dojo_env_reset(self.h, C.byref(spec), int(B), _p(s0), _p(mask), _p(dS)), "dojo_env_reset")
            return None
        assert S.flags.c_contiguous and S.dtype == np.float64
        if mask is not None:
            mask = np.ascontiguousarray(mask, dtype=np.int32)
        self._check(self.L.dojo_env_reset(self.h, C.byref(spec), S.shape[0], _p(s0), _p(mask), _p(S)), "dojo_env_reset")
        return S

    # ------------------------------------------------------------------ device buffers (resident data)
    def step_device(self, dZ: int, dU: Optional[int], dZn: int, B: int, opts=None, dstatus: Optional[int] = None, diters: Optional[int] = None,
                    dsol: Optional[int] = None, dfext: Optional[int] = None, flags: int = 0, stream: int = 0, dtrace: Optional[int] = None):
        """dojo_step_async on device pointers; with dtrace ([B, max_iter, 5] doubles) the traced step, dojo_step_trace_async."""
        o = opts if opts is not None else capi.solver_options()
        if dtrace is not None:
            rc = self.L.dojo_step_trace_async(self.h, C.byref(o), int(B), _p(dZ), _p(dU), _p(dfext), _p(dZn), _p(dsol), _p(dstatus), _p(diters),
                                              _p(dtrace), flags, C.c_void_p(int(stream)))
            self._check(rc, "dojo_step_trace_async")
            return
        rc = self.L.dojo_step_async(self.h, C.byref(o), int(B), _p(dZ), _p(dU), _p(dfext), _p(dZn), _p(dsol), _p(dstatus), _p(diters), flags,
                                    C.c_void_p(int(stream)))
        self._check(rc, "dojo_step_async")

    def minimal_to_maximal_device(self, dX: int, dZ: int, B: int, stream: int = 0):
        self._check(self.L.dojo_minimal_to_maximal_async(self.h, int(B), _p(dX), _p(dZ), C.c_void_p(int(stream))), "dojo_minimal_to_maximal_async")

    def maximal_to_minimal_device(self, dZ: int, dX: int, B: int, stream: int = 0):
        self._check(self.L.dojo_maximal_to_minimal_async(self.h, int(B), _p(dZ), _p(dX), C.c_void_p(int(stream))), "dojo_maximal_to_minimal_async")

    def maximal_to_minimal_jacobian_device(self, dZ: int, dJ: int, B: int, stream: int = 0):
        self._check(self.L.dojo_maximal_to_minimal_jacobian_async(self.h, int(B), _p(dZ), _p(dJ), C.c_void_p(int(stream))), "dojo_maximal_to_minimal_jacobian_async")

    def minimal_to_maximal_jacobian_device(self, dZ: int, dJ: int, B: int, stream: int = 0):
        self._check(self.L.dojo_minimal_to_maximal_jacobian_async(self.h, int(B), _p(dZ), _p(dJ), C.c_void_p(int(stream))), "dojo_minimal_to_maximal_jacobian_async")

    def minimal_gradients_device(self, dX: int, dU: Optional[int], dXn: int, dGx: int, dGu: int, B: int, opts=None, dstatus=None, diters=None):
        """device-resident get_minimal_gradients! (synchronises the handle's stream before returning)"""
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_minimal_gradients(self.h, C.byref(o), int(B), _p(dX), _p(dU), _p(dXn), _p(dGx), _p(dGu), _p(dstatus), _p(diters))
        self._check(rc, "dojo_minimal_gradients")

    def rollout_device(self, dZ0: int, dU: Optional[int], dZf: int, B: int, T: int, opts=None, dtraj: Optional[int] = None, dstatus: Optional[int] = None,
                       stream: int = 0):
        """T steps fused in one launch on resident data (U is [T, B, nu] on the device)."""
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_rollout_async(self.h, C.byref(o), int(B), int(T), _p(dZ0), _p(dU), _p(dZf), _p(dtraj), _p(dstatus), C.c_void_p(int(stream)))
        self._check(rc, "dojo_rollout_async")

    def step_grad_device(self, dZ: int, dU: Optional[int], dZn: int, dFz: int, dFu: int, B: int, opts=None, dstatus=None, diters=None, flags: int = 0,
                         stream: int = 0):
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_step_grad_async(self.h, C.byref(o), int(B), _p(dZ), _p(dU), None, _p(dZn), _p(dFz), _p(dFu), _p(dstatus), _p(diters), flags,
                                         C.c_void_p(int(stream)))
        self._check(rc, "dojo_step_grad_async")

    def rollout_grad_device(self, dZ0: int, dU: Optional[int], dZ_traj: int, dFz: int, dFu: int, B: int, T: int, opts=None, dstatus=None,
                            diters=None, stream: int = 0):
        """dojo_rollout_grad_async on device pointers: Z_traj [T+1, B, 13Nb], Fz [T, B, 12Nb, 12Nb] and Fu [T, B, nu, 12Nb] (column-major
        per pair), status / iters [T, B]; dZ0 may be dZ_traj (slab 0 already holds Z0)."""
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_rollout_grad_async(self.h, C.byref(o), int(B), int(T), _p(dZ0), _p(dU), _p(dZ_traj), _p(dFz), _p(dFu), _p(dstatus),
                                            _p(diters), C.c_void_p(int(stream)))
        self._check(rc, "dojo_rollout_grad_async")

    def rollout_feedback_device(self, dZ0: int, dZf: int, B: int, T: int, dK: int, steps: int = 1, envs: int = 1, dK_i=None, dx_ref=None, du_ref=None,
                                dxi=None, dtraj=None, dU_applied=None, dstatus=None, opts=None, stream: int = 0):
        """dojo_rollout_feedback_async on device pointers: K / K_i [steps, envs, 2nu, nu] (column-major [nu x 2nu] per entry), x_ref
        [steps, envs, 2nu], u_ref [steps, envs, nu], xi [B, 2nu] in/out, Z_traj [T, B, 13Nb], U_applied [T, B, nu], status [B]."""
        o = opts if opts is not None else capi.solver_options()
        cp = lambda d: None if d is None else C.cast(C.c_void_p(int(d)), capi.c_double_p)
        fb = capi.DojoFeedback(int(steps), int(envs), cp(dK), cp(dK_i), cp(dx_ref), cp(du_ref))
        rc = self.L.dojo_rollout_feedback_async(self.h, C.byref(o), int(B), int(T), _p(dZ0), C.byref(fb), _p(dxi), _p(dZf), _p(dtraj), _p(dU_applied),
                                                _p(dstatus), C.c_void_p(int(stream)))
        self._check(rc, "dojo_rollout_feedback_async")

    def lqr_backward_device(self, B: int, T: int, dX_traj: int, dGx: int, dGu: int, dK: int, dk: int, dQ: int, dR: int, dQ_final: int,
                            steps: int = 1, envs: int = 1, dx_goal=None, du_goal=None, dx_goal_final=None, dU=None, dmu=None, active=None,
                            ddV=None, dstatus=None, stream: int = 0):
        """dojo_lqr_backward_async on device pointers, in the layouts of dojo_rollout_minimal_gradients: X_traj [T+1, B, 2nu], Gx / Gu
        column-major per pair ([T, B, 2nu, 2nu] / [T, B, nu, 2nu] in memory), K out [T, B, 2nu, nu] in memory (column-major [nu x 2nu]),
        k [T, B, nu], dV [B, 2], status [B]; the cost arrays as cost_arrays returns them; active: a host [nu] mask or None."""
        cp = lambda d: None if d is None else C.cast(C.c_void_p(int(d)), capi.c_double_p)
        c = capi.DojoQuadraticCost(int(steps), int(envs), cp(dQ), cp(dR), cp(dx_goal), cp(du_goal), cp(dQ_final), cp(dx_goal_final))
        act = None if active is None else np.ascontiguousarray(np.asarray(active).astype(np.int32).reshape(self.nu))
        rc = self.L.dojo_lqr_backward_async(self.h, int(B), int(T), C.byref(c), _p(act), _p(dX_traj), _p(dU), _p(dGx), _p(dGu), _p(dmu), _p(dK),
                                            _p(dk), _p(ddV), _p(dstatus), C.c_void_p(int(stream)))
        self._check(rc, "dojo_lqr_backward_async")

    # ---- multi-GPU: the exchange of the next states fused into the step (include/dojo_b200.h, SURVEY.md 8e)
    def gather_create(self, world: int, rank: int, B_local: int):
        g = C.c_void_p()
        self._check(self.L.dojo_gather_create(self.h, int(world), int(rank), int(B_local), C.byref(g)), "dojo_gather_create")
        return g

    def gather_export(self, g) -> bytes:
        buf = C.create_string_buffer(128)
        self._check(self.L.dojo_gather_export(g, buf), "dojo_gather_export")
        return buf.raw

    def gather_connect(self, g, all_handles: bytes):
        buf = C.create_string_buffer(all_handles, len(all_handles))
        self._check(self.L.dojo_gather_connect(g, buf), "dojo_gather_connect")

    def gather_buffer(self, g) -> int:
        return int(self.L.dojo_gather_buffer(g) or 0)

    def gather_destroy(self, g):
        self.L.dojo_gather_destroy(g)

    def step_gather_device(self, g, dZ: int, dU: Optional[int], dZn: int, B: int, opts=None, dstatus=None, diters=None, flags: int = 0, stream: int = 0):
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_step_gather_async(self.h, g, C.byref(o), int(B), _p(dZ), _p(dU), None, _p(dZn), _p(dstatus), _p(diters), flags, C.c_void_p(int(stream)))
        self._check(rc, "dojo_step_gather_async")

    def step_grad_gather_device(self, g, dZ: int, dU: Optional[int], dZn: int, dFz: int, dFu: int, B: int, opts=None, dstatus=None, diters=None, flags: int = 0,
                                stream: int = 0):
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.dojo_step_grad_gather_async(self.h, g, C.byref(o), int(B), _p(dZ), _p(dU), None, _p(dZn), _p(dFz), _p(dFu), _p(dstatus), _p(diters), flags,
                                                C.c_void_p(int(stream)))
        self._check(rc, "dojo_step_grad_gather_async")
