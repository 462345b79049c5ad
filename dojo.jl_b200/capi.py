"""ctypes mirror of include/dojo_b200.h (struct layouts + flattening of a Mechanism).

Interface definitions only -- no compute.  Used by the product binding (solver.py) and, for the
struct layouts, by the oracle's test wrapper (oracle/oracle.py).
"""
import ctypes as C

import numpy as np

from .mechanism import Mechanism

c_double_p = C.POINTER(C.c_double)
c_int32_p = C.POINTER(C.c_int32)


class DojoBodyDesc(C.Structure):
    _fields_ = [("mass", C.c_double), ("inertia", C.c_double * 9)]


class DojoJointElementDesc(C.Structure):
    _fields_ = [("nlambda", C.c_int32), ("nlimits", C.c_int32), ("axis_mask", C.c_double * 9),
                ("spring", C.c_double), ("damper", C.c_double), ("spring_offset", C.c_double * 3),
                ("limit_lo", C.c_double * 3), ("limit_hi", C.c_double * 3)]


class DojoJointDesc(C.Structure):
    _fields_ = [("parent_body", C.c_int32), ("child_body", C.c_int32), ("vertex_parent", C.c_double * 3),
                ("vertex_child", C.c_double * 3), ("orientation_offset", C.c_double * 4),
                ("tra", DojoJointElementDesc), ("rot", DojoJointElementDesc)]


class DojoContactDesc(C.Structure):
    _fields_ = [("type", C.c_int32), ("parent_body", C.c_int32), ("friction_coefficient", C.c_double),
                ("tangent", C.c_double * 6), ("normal", C.c_double * 3), ("origin", C.c_double * 3),
                ("radius", C.c_double), ("offset", C.c_double * 3)]


class DojoMechanismDesc(C.Structure):
    _fields_ = [("num_bodies", C.c_int32), ("num_joints", C.c_int32), ("num_contacts", C.c_int32),
                ("timestep", C.c_double), ("input_scaling", C.c_double), ("gravity", C.c_double * 3),
                ("bodies", C.POINTER(DojoBodyDesc)), ("joints", C.POINTER(DojoJointDesc)),
                ("contacts", C.POINTER(DojoContactDesc))]


class DojoSolverOptions(C.Structure):
    """SolverOptions (src/solver/options.jl:16-26), same defaults."""
    _fields_ = [("rtol", C.c_double), ("btol", C.c_double), ("ls_scale", C.c_double), ("max_iter", C.c_int32),
                ("max_ls", C.c_int32), ("undercut", C.c_double), ("no_progress_max", C.c_int32),
                ("no_progress_undercut", C.c_double), ("verbose", C.c_int32)]


class DojoEnvSpec(C.Structure):
    """Environment layer (include/dojo_b200.h: DojoEnvSpec)."""
    _fields_ = [("n_unactuated", C.c_int32), ("contact_obs", C.c_int32), ("forward_index", C.c_int32), ("healthy_index", C.c_int32),
                ("bound_index", C.c_int32), ("w_forward", C.c_double), ("w_control", C.c_double), ("w_contact", C.c_double),
                ("survive_reward", C.c_double), ("healthy_min", C.c_double), ("healthy_max", C.c_double), ("bound_abs", C.c_double)]


class DojoFeedback(C.Structure):
    """Closed-loop rollout law (include/dojo_b200.h: DojoFeedback): u_t = u_ref - K (x_t - x_ref) - K_i xi_t on the minimal state.
    Every array holds steps (1 or T) x envs (1 or B) entries; K and K_i are column-major [nu x 2nu] per entry."""
    _fields_ = [("steps", C.c_int32), ("envs", C.c_int32), ("K", c_double_p), ("K_i", c_double_p), ("x_ref", c_double_p), ("u_ref", c_double_p)]


class DojoFeedbackGrad(C.Structure):
    """Law gradients of dojo_rollout_feedback_vjp (include/dojo_b200.h: DojoFeedbackGrad), each nullable and always per environment:
    [.. x B x steps] with the DojoFeedback's steps; K / K_i column-major [nu x 2nu] per entry."""
    _fields_ = [("K", c_double_p), ("K_i", c_double_p), ("x_ref", c_double_p), ("u_ref", c_double_p)]


class DojoQuadraticCost(C.Structure):
    """Quadratic tracking cost of dojo_lqr_backward (include/dojo_b200.h: DojoQuadraticCost).  Q, R, x_goal, u_goal hold steps (1 or T) x
    envs (1 or B) entries, Q_final and x_goal_final envs entries; matrices column-major per entry."""
    _fields_ = [("steps", C.c_int32), ("envs", C.c_int32), ("Q", c_double_p), ("R", c_double_p), ("x_goal", c_double_p), ("u_goal", c_double_p),
                ("Q_final", c_double_p), ("x_goal_final", c_double_p)]


def quadratic_cost(steps, envs, Q, R, x_goal=None, u_goal=None, Q_final=None, x_goal_final=None) -> DojoQuadraticCost:
    """a DojoQuadraticCost over host arrays (solver.cost_arrays's output); the arrays must outlive the struct"""
    p = lambda a: None if a is None else dptr(a)
    return DojoQuadraticCost(int(steps), int(envs), p(Q), p(R), p(x_goal), p(u_goal), p(Q_final), p(x_goal_final))


def env_spec(n_unactuated=0, contact_obs=False, forward_index=-1, healthy_index=-1, bound_index=-1, w_forward=0.0, w_control=0.0,
             w_contact=0.0, survive_reward=0.0, healthy_min=-float("inf"), healthy_max=float("inf"), bound_abs=float("inf")) -> DojoEnvSpec:
    return DojoEnvSpec(int(n_unactuated), int(bool(contact_obs)), int(forward_index), int(healthy_index), int(bound_index), float(w_forward),
                       float(w_control), float(w_contact), float(survive_reward), float(healthy_min), float(healthy_max), float(bound_abs))


def solver_options(rtol=1.0e-6, btol=1.0e-4, ls_scale=0.5, max_iter=50, max_ls=10, undercut=float("inf"),
                   no_progress_max=3, no_progress_undercut=10.0, verbose=False) -> DojoSolverOptions:
    return DojoSolverOptions(rtol, btol, ls_scale, max_iter, max_ls, undercut, no_progress_max,
                             no_progress_undercut, int(verbose))


def _fill(arr, values):
    v = np.asarray(values, dtype=float).reshape(-1)
    for i in range(len(v)):
        arr[i] = float(v[i])


def _element(e) -> DojoJointElementDesc:
    d = DojoJointElementDesc()
    d.nlambda, d.nlimits = e.nlambda, e.nlimits
    _fill(d.axis_mask, e.axis_mask)
    d.spring, d.damper = float(e.spring), float(e.damper)
    _fill(d.spring_offset, e.spring_offset)
    if e.nlimits:
        if e.nlimits != 3 - e.nlambda:
            raise ValueError("joint limits must cover every free axis of the element (joints/limits.jl)")
        _fill(d.limit_lo, e.limit_lo)
        _fill(d.limit_hi, e.limit_hi)
    return d


def flatten(mech: Mechanism):
    """Mechanism -> (DojoMechanismDesc, keepalive).  The caller must keep `keepalive` referenced
    while the descriptor is in use (dojo_create copies it)."""
    bodies = (DojoBodyDesc * max(mech.Nb, 1))()
    for i, b in enumerate(mech.bodies):
        bodies[i].mass = float(b.mass)
        _fill(bodies[i].inertia, b.inertia)
    joints = (DojoJointDesc * max(mech.Ne, 1))()
    for i, j in enumerate(mech.joints):
        joints[i].parent_body, joints[i].child_body = int(j.parent), int(j.child)
        _fill(joints[i].vertex_parent, j.vertex_parent)
        _fill(joints[i].vertex_child, j.vertex_child)
        _fill(joints[i].orientation_offset, j.orientation_offset)
        joints[i].tra = _element(j.tra)
        joints[i].rot = _element(j.rot)
    contacts = (DojoContactDesc * max(mech.Ni, 1))()
    for i, c in enumerate(mech.contacts):
        contacts[i].type = int(getattr(c, "type", 2))
        contacts[i].parent_body = int(c.body)
        contacts[i].friction_coefficient = float(c.friction)
        _fill(contacts[i].tangent, c.tangent)
        _fill(contacts[i].normal, c.normal)
        _fill(contacts[i].origin, c.origin)
        contacts[i].radius = float(c.radius)
        _fill(contacts[i].offset, c.offset)
    d = DojoMechanismDesc()
    d.num_bodies, d.num_joints, d.num_contacts = mech.Nb, mech.Ne, mech.Ni
    d.timestep, d.input_scaling = mech.timestep, mech.input_scaling
    _fill(d.gravity, mech.gravity)
    d.bodies = C.cast(bodies, C.POINTER(DojoBodyDesc))
    d.joints = C.cast(joints, C.POINTER(DojoJointDesc))
    d.contacts = C.cast(contacts, C.POINTER(DojoContactDesc))
    return d, (bodies, joints, contacts)


def dptr(a: np.ndarray):
    return a.ctypes.data_as(c_double_p)


def iptr(a: np.ndarray):
    return a.ctypes.data_as(c_int32_p)
