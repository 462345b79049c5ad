"""Host-side mirror of the reference interface for the hot path (same names, argument meaning and error behaviour;
Python has no `!`, so `step!` is `step`):

    reference (Julia)                                              here
    -------------------------------------------------------------  ------------------------------------------
    SolverOptions{T}(; rtol, btol, ...)   solver/options.jl:16-26   SolverOptions(rtol=..., btol=..., ...)
    step!(mechanism, z, u; opts)          simulation/step.jl:11     step(mechanism, z, u, opts=None)
    simulate!(mechanism, steps, storage, control!; opts)            simulate(mechanism, steps, control=None, record=False, opts=None)
                                          simulation/simulate.jl:16
    controller! reading get_minimal_state (examples/control)        simulate(..., control=LinearFeedback(K, x_ref, u_ref, K_i, xi))
    get_maximal_gradients!(mechanism, z, u; opts)                   get_maximal_gradients(mechanism, z, u, opts=None)
                                          gradients/state.jl:69
    get_contact_gradients(mechanism)      gradients/contact.jl:1    get_contact_gradients(mechanism, z, u, opts=None)
    simulate! + get_maximal_gradients! at every step                get_trajectory_gradients(mechanism, z0, U, opts=None)
    simulate! + get_minimal_gradients! at every step                get_minimal_trajectory_gradients(mechanism, x0, U, opts=None)
    mehrotra!(mechanism; opts) -> :success / :failed                status codes returned next to the states (STATUS)
    minimal_to_maximal(mechanism, x)      mechanism/state.jl:9      minimal_to_maximal(mechanism, x)
    maximal_to_minimal(mechanism, z)      mechanism/state.jl:44     maximal_to_minimal(mechanism, z)
    step_minimal_coordinates!(mechanism, x, u; opts)                step_minimal_coordinates(mechanism, x, u, opts=None)
                                          simulation/step.jl:42
    maximal_to_minimal_jacobian(mechanism, z)  gradients/state.jl:9   maximal_to_minimal_jacobian(mechanism, z)
    minimal_to_maximal_jacobian(mechanism, x)  gradients/state.jl:136 minimal_to_maximal_jacobian(mechanism, x)
    get_minimal_gradients!(mechanism, x, u; opts)                   get_minimal_gradients(mechanism, x, u, opts=None)
                                          gradients/state.jl:182
    IterativeLQR.jl (docs/src/examples/trajectory_optimization.md)  ilqr(mechanism, x0, U0, QuadraticCost(Q, R, ...), iterations)
    simulate!(...; record=true) -> Storage  simulation/simulate.jl:16, storage.jl:15-67      simulate_record(mechanism, steps, ...) -> Storage
    momentum / kinetic_energy / potential_energy / mechanical_energy(mechanism, storage)   same names (mechanics/{momentum,energy}.jl)

NEW relative to the reference: every function also accepts a batch -- z of shape [B, 13 Nb], u of shape [B, nu] --
and then returns batched results.  All compute happens in libdojo_b200.so on the GPU (solver.BatchedStepper).

Deviations (documented switches, SURVEY.md Appendix D):
  * step returns the TRUE next state (x3, v25, q3, w25) -- the mechanism's internal state after step! -- unless
    literal_q1=True (the reference's return value advances the configuration twice, Q1);
  * gradients are the consistent IFT gradients at the solution unless literal_q2=True (get_maximal_gradients! builds the data
    Jacobian AFTER update_state! but solves against the KKT matrix assembled before it, Q2);
  * "Excessive angular velocity" (solver/line_search.jl:18-20): status code 2 is reserved for it, but the reference's test can
    never fire -- candidate_step! clips |w|^2 to (3.9/h^2)^2 / |w|^2 < 3.9/h^2 before line_search! compares it with 3.91/h^2
    (DESIGN.md section 6) -- so no path produces it; _check_single keeps the mapping to the reference's error().
"""
import math
import warnings
from typing import Callable, Optional

import numpy as np

from . import capi
from .mechanism import Mechanism
from .solver import DOJO_FLAG_Q1_LITERAL_RETURN, DOJO_FLAG_Q2_LITERAL_GRADIENTS, DOJO_FLAG_Q17_LITERAL_INPUT_JACOBIAN, STATUS, BatchedStepper, cost_arrays

SolverOptions = capi.solver_options

_steppers = {}


def _stepper(mech: Mechanism, B: int, device: int = 0) -> BatchedStepper:
    key = (id(mech), device)
    s = _steppers.get(key)
    if s is None or s.max_batch < B:
        if s is not None:
            s.close()
        s = BatchedStepper(mech, max(B, 64), device)
        _steppers[key] = s
    return s


def _check_single(status):
    if int(status[0]) == 2:
        raise RuntimeError("Excessive angular velocity.")  # reference: error(...) in line_search!


def _scn(a: float) -> str:
    """scn(a, digits=0) (utilities/methods.jl:9-43): one significant digit and the exponent, e.g. ' 4e-5'."""
    a = float(a)
    if math.isnan(a):
        return " NaN "
    if a == math.inf:
        return " Inf"
    if a == -math.inf:
        return "-Inf"
    if a == 0:
        e, m = 0, 0.0
    else:
        e = int(math.floor(math.log(abs(a)) / math.log(10)))
        m = a * math.exp(-e * math.log(10))
    m = float(round(m))  # Julia's round: to nearest, ties to even, like Python's
    if m == 10.0:
        m, e = 1.0, e + 1
    sgn = " " if a >= 0 else ""
    return f"{sgn}{int(math.floor(m))}e{'+' if e >= 0 else '-'}{abs(e)}"


def format_solver_trace(trace) -> str:
    """The table mehrotra! prints with SolverOptions(verbose = true) (solver_header / solver_status, solver/mehrotra.jl:75-98) for one
    solve, from its trace [max_iter, 5] (BatchedStepper.step(..., trace=True)): one line per loop head n, `n  bvio  rvio  α  μ`, where α
    and μ belong to the iteration before the head.  The reference's last two columns, |res|∞ and |Δ|∞, are left out: there both are
    norm(full_vector(system), Inf) of the same vector, so they print the same number, and that vector -- the residual assembled at the
    iterate of the head -- is never formed on the device, which decides convergence from the violations alone."""
    tr = np.asarray(trace, dtype=float)
    rows = int(np.count_nonzero(~np.isnan(tr[:, 4]))) if tr.size else 0  # the trials column is NaN exactly in the padding rows
    lines = [" " * 49, "n    bvio    rvio     α       μ", "–" * 49]
    for r in range(rows):
        rvio, bvio, alpha, mu = tr[r, :4]
        lines.append(f"{r + 1}   {_scn(bvio)}   {_scn(rvio)}   {_scn(alpha)}   {_scn(mu)}")
    return "\n".join(lines)


def _print_trace(trace, status) -> None:
    print(format_solver_trace(trace))
    if int(status) == 1:
        warnings.warn("failed mehrotra")  # solver/mehrotra.jl:31, at the head of the last iteration


def _verbose(opts) -> bool:
    return opts is not None and bool(opts.verbose)


def step(mechanism: Mechanism, z, u, opts=None, literal_q1: bool = False, device: int = 0):
    """step!(mechanism, z, u; opts).  z: [13Nb] or [B, 13Nb]; u: [nu] or [B, nu].  Returns z_next (same shape); for a batch
    also (status, iters).  With opts.verbose and a single environment the step runs traced and prints the solver's table
    (format_solver_trace) and, when it ends :failed, the warning "failed mehrotra", as mehrotra! does; batched calls do not print
    (use BatchedStepper.step(..., trace=True) for the traces of a batch)."""
    z = np.asarray(z, dtype=float)
    single = z.ndim == 1
    Z = np.atleast_2d(z)
    U = np.atleast_2d(np.asarray(u, dtype=float))
    s = _stepper(mechanism, Z.shape[0], device)
    flags = DOJO_FLAG_Q1_LITERAL_RETURN if literal_q1 else 0
    if single and _verbose(opts):
        Zn, status, iters, tr = s.step(Z, U, opts, flags=flags, trace=True)
        _print_trace(tr[0], status[0])
    else:
        Zn, status, iters = s.step(Z, U, opts, flags=flags)
    if single:
        _check_single(status)
        return Zn[0]
    return Zn, status, iters


class LinearFeedback:
    """A controller! that reads the minimal state at every step (get_minimal_state, examples/control) and applies the time-varying
    affine law  u_t = u_ref - K (x_t - x_ref) - K_i xi_t,  xi_t = xi_{t-1} + h (x_t - x_ref)  (the integral is updated before use, as
    pendulum_pid.jl does).  K, K_i [nu, 2nu], x_ref [2nu], u_ref [nu], each optionally per environment ([B, ...]) or per step and
    environment ([steps, 1 or B, ...]); K_i None: no integral term.  simulate(..., control=LinearFeedback(...)) evaluates the law inside
    the fused rollout on the device and updates `xi` ([2nu], or [B, 2nu]), so that a second call continues the integral.
    Examples: pendulum_pid.jl is K = [Kp Kd], K_i = [Ki 0], x_ref = [pi/2, 0]; cartpole_lqr.jl is an LQR row on the cart input."""

    def __init__(self, K, x_ref=None, u_ref=None, K_i=None, xi=None):
        self.K, self.x_ref, self.u_ref, self.K_i = K, x_ref, u_ref, K_i
        self.xi = None if xi is None else np.array(xi, dtype=float)


def simulate(mechanism: Mechanism, steps: int, z0=None, control: Optional[Callable] = None, record: bool = False, opts=None, device: int = 0):
    """simulate!(mechanism, steps, storage, control!): `control(k)` returns the input(s) of step k ([nu] or [B, nu]; None = 0).
    Returns the final state(s) and, with record=True, the trajectory [steps, B, 13Nb] (the reference's Storage).
    The steps are fused into one launch, except with opts.verbose and a single environment: then every step is its own traced
    launch and prints its solver table, as simulate! does with verbose = true (same results).  Batched calls do not print.
    control = LinearFeedback(...) closes the loop on the device: the law is evaluated at every step on the state the step starts from,
    in the same single launch (opts.verbose is refused: a traced closed loop is not provided)."""
    z0 = mechanism.z0 if z0 is None else z0
    z0 = np.asarray(z0, dtype=float)
    single = z0.ndim == 1
    Z = np.atleast_2d(z0)
    B = Z.shape[0]
    s = _stepper(mechanism, B, device)
    if isinstance(control, LinearFeedback):
        if _verbose(opts):
            raise ValueError("simulate: opts.verbose with a LinearFeedback controller is not supported (the traced step runs open loop)")
        fb = control
        Zf, _, traj, _, xi = s.rollout_feedback(Z, steps, fb.K, fb.x_ref, fb.u_ref, fb.K_i, fb.xi, opts, record=record)
        if xi is not None:
            new = xi[0] if (single and (fb.xi is None or np.ndim(fb.xi) == 1)) else xi
            if fb.xi is not None and np.shape(fb.xi) == new.shape:
                fb.xi[...] = new
            else:
                fb.xi = new
        if single:
            return (Zf[0], traj[:, 0]) if record else Zf[0]
        return (Zf, traj) if record else Zf
    U = None
    if control is not None:
        U = np.zeros((steps, B, mechanism.nu))
        for k in range(steps):
            uk = control(k)
            if uk is not None:
                U[k] = np.asarray(uk, dtype=float)
    if single and _verbose(opts):
        traj = np.empty((steps, B, mechanism.nz)) if record else None
        Zf = Z
        for k in range(steps):
            Zf, status, _, tr = s.step(Zf, None if U is None else U[k], opts, trace=True)
            _print_trace(tr[0], status[0])
            if record:
                traj[k] = Zf
    else:
        out = s.rollout(Z, U, steps, opts, record=record)
        Zf, traj = out[0], (out[2] if record else None)
    if single:
        return (Zf[0], traj[:, 0]) if record else Zf[0]
    return (Zf, traj) if record else Zf


def get_maximal_gradients(mechanism: Mechanism, z, u, opts=None, device: int = 0, literal_q2: bool = False, literal_q17: bool = False):
    """get_maximal_gradients!(mechanism, z, u; opts) -> (jacobian_state [12Nb x 12Nb], jacobian_control [12Nb x nu]);
    batched inputs give [B, 12Nb, 12Nb] and [B, 12Nb, nu].  literal_q2=True reproduces the reference's literal result (data
    Jacobian and chain rule at the state shifted by update_state!, gradients/state.jl:69-76); the default is the consistent
    implicit-function-theorem gradient.  literal_q17=True leaves d(input impulse)/d(configuration) out of the data Jacobian, as
    gradients/data.jl does; the reference's get_maximal_gradients! is literal_q2=literal_q17=True."""
    z = np.asarray(z, dtype=float)
    single = z.ndim == 1
    Z = np.atleast_2d(z)
    U = np.atleast_2d(np.asarray(u, dtype=float))
    s = _stepper(mechanism, Z.shape[0], device)
    flags = (DOJO_FLAG_Q2_LITERAL_GRADIENTS if literal_q2 else 0) | (DOJO_FLAG_Q17_LITERAL_INPUT_JACOBIAN if literal_q17 else 0)
    _, Fz, Fu, status, _ = s.step_grad(Z, U, opts, flags=flags)
    if single:
        _check_single(status)
        return Fz[0], Fu[0]
    return Fz, Fu


def get_contact_gradients(mechanism: Mechanism, z, u, opts=None, device: int = 0):
    """get_contact_gradients!(mechanism, z, u; opts) (gradients/contact.jl:1-55, the step is taken first as in
    get_maximal_gradients!) -> (jacobian_state [12Nb x 12Nb], jacobian_contact [12Nb x 5Ni]); per contact the data are
    [friction_coefficient, contact_radius, contact_origin(3)].  Batched inputs give [B, ...]."""
    z = np.asarray(z, dtype=float)
    single = z.ndim == 1
    Z = np.atleast_2d(z)
    U = np.atleast_2d(np.asarray(u, dtype=float))
    _, Fz, _, Fc, status, _ = _stepper(mechanism, Z.shape[0], device).step_grad_contact(Z, U, opts)
    if single:
        _check_single(status)
        return Fz[0], Fc[0]
    return Fz, Fc


def _trajectory_inputs(x0, U):
    x0 = np.asarray(x0, dtype=float)
    single = x0.ndim == 1
    X0 = np.atleast_2d(x0)
    U = np.asarray(U, dtype=float)
    if single:
        U = U.reshape(U.shape[0], 1, -1)
    return single, X0, np.ascontiguousarray(U), U.shape[0]


def get_trajectory_gradients(mechanism: Mechanism, z0, U, opts=None, device: int = 0):
    """simulate!(mechanism, T, ...) from z0 with the open-loop inputs U and get_maximal_gradients! at every step, fused on the device:
    z0 [13Nb], U [T, nu] -> (Z_traj [T+1, 13Nb] with Z_traj[0] = z0, Fz [T, 12Nb, 12Nb] = dz_{t+1}/dz_t, Fu [T, 12Nb, nu] = dz_{t+1}/du_t,
    status [T] of every step).  Batched: z0 [B, 13Nb], U [T, B, nu] -> [T+1, B, ...], [T, B, ...], status [T, B]."""
    single, Z0, U, T = _trajectory_inputs(z0, U)
    traj, Fz, Fu, status, _ = _stepper(mechanism, Z0.shape[0], device).rollout_grad(Z0, U, T, opts)
    if single:
        return traj[:, 0], Fz[:, 0], Fu[:, 0], status[:, 0]
    return traj, Fz, Fu, status


def get_minimal_trajectory_gradients(mechanism: Mechanism, x0, U, opts=None, device: int = 0):
    """get_trajectory_gradients in minimal coordinates (get_minimal_gradients! at every step): x0 [2nu], U [T, nu] -> (X_traj [T+1, 2nu],
    Gx [T, 2nu, 2nu], Gu [T, 2nu, nu], status [T]).  The rollout runs in maximal coordinates from minimal_to_maximal(x0); X_traj is its
    trajectory mapped to minimal coordinates.  Batched: x0 [B, 2nu], U [T, B, nu]."""
    single, X0, U, T = _trajectory_inputs(x0, U)
    Xt, Gx, Gu, status, _ = _stepper(mechanism, X0.shape[0], device).rollout_minimal_gradients(X0, U, T, opts)
    if single:
        return Xt[:, 0], Gx[:, 0], Gu[:, 0], status[:, 0]
    return Xt, Gx, Gu, status


def minimal_to_maximal(mechanism: Mechanism, x, device: int = 0):
    """minimal_to_maximal(mechanism, x): x [2 nu] or [B, 2 nu] (per joint [c_tra; c_rot; v_tra; v_rot]) -> z [13 Nb] / [B, 13 Nb]."""
    x = np.asarray(x, dtype=float)
    X = np.atleast_2d(x)
    Z = _stepper(mechanism, X.shape[0], device).minimal_to_maximal(X)
    return Z[0] if x.ndim == 1 else Z


def maximal_to_minimal(mechanism: Mechanism, z, device: int = 0):
    """maximal_to_minimal(mechanism, z): z [13 Nb] or [B, 13 Nb] -> x [2 nu] / [B, 2 nu]."""
    z = np.asarray(z, dtype=float)
    Z = np.atleast_2d(z)
    X = _stepper(mechanism, Z.shape[0], device).maximal_to_minimal(Z)
    return X[0] if z.ndim == 1 else X


def step_minimal_coordinates(mechanism: Mechanism, x, u, opts=None, device: int = 0, literal: bool = False):
    """step_minimal_coordinates!(mechanism, x, u; opts) -> x_next (what DojoEnvironments.step! calls); for a batch also
    (status, iters).  The maximal states stay on the device between the three launches.  literal = True returns what the reference
    literally returns (step!'s return value advances the configuration a second time, SURVEY.md Q1) instead of the state after the step."""
    x = np.asarray(x, dtype=float)
    single = x.ndim == 1
    X = np.atleast_2d(x)
    U = np.atleast_2d(np.asarray(u, dtype=float))
    Xn, status, iters = _stepper(mechanism, X.shape[0], device).step_minimal(X, U, opts, flags=1 if literal else 0)
    if single:
        _check_single(status)
        return Xn[0]
    return Xn, status, iters


def maximal_to_minimal_jacobian(mechanism: Mechanism, z, device: int = 0):
    """maximal_to_minimal_jacobian(mechanism, z) -> [2 nu x 12 Nb] (columns: attitude-reduced [x, v, phi, w] per body);
    batched z gives [B, 2 nu, 12 Nb]."""
    z = np.asarray(z, dtype=float)
    Z = np.atleast_2d(z)
    J = _stepper(mechanism, Z.shape[0], device).maximal_to_minimal_jacobian(Z)
    return J[0] if z.ndim == 1 else J


def minimal_to_maximal_jacobian(mechanism: Mechanism, x, device: int = 0):
    """minimal_to_maximal_jacobian(mechanism, x) -> [12 Nb x 2 nu], the derivative of minimal_to_maximal at x (the
    reference reads the mechanism's stored state, which its callers set to minimal_to_maximal(x) first; it chains the
    partials in mechanism.bodies order, identical to the root -> leaves order used here when parents precede children)."""
    x = np.asarray(x, dtype=float)
    X = np.atleast_2d(x)
    s = _stepper(mechanism, X.shape[0], device)
    J = s.minimal_to_maximal_jacobian(s.minimal_to_maximal(X))
    return J[0] if x.ndim == 1 else J


def get_minimal_gradients(mechanism: Mechanism, x, u, opts=None, device: int = 0):
    """get_minimal_gradients!(mechanism, x, u; opts) -> (minimal_jacobian_state [2nu x 2nu], minimal_jacobian_control
    [2nu x nu]); batched inputs give [B, 2nu, 2nu] and [B, 2nu, nu].  Consistent variant (SURVEY Q2): the map Jacobians are
    taken at z = minimal_to_maximal(x) and at the true next state."""
    x = np.asarray(x, dtype=float)
    single = x.ndim == 1
    X = np.atleast_2d(x)
    U = np.atleast_2d(np.asarray(u, dtype=float))
    _, Gx, Gu, status, _ = _stepper(mechanism, X.shape[0], device).minimal_gradients(X, U, opts)
    if single:
        _check_single(status)
        return Gx[0], Gu[0]
    return Gx, Gu


class QuadraticCost:
    """The quadratic tracking cost of trajectory optimisation in minimal coordinates (dojo_lqr_backward's DojoQuadraticCost):
        J = sum_t 1/2 (x_t - xg_t)' Q_t (x_t - xg_t) + 1/2 (u_t - ug_t)' R_t (u_t - ug_t)  +  1/2 (x_T - xg_T)' Q_final (x_T - xg_T).
    Q [2nu, 2nu], R [nu, nu], x_goal [2nu], u_goal [nu], each also per environment [B, ...] or per step [T, 1 or B, ...]; Q_final and
    x_goal_final also [B, ...].  Defaults: goals 0, Q_final = the last step's Q, x_goal_final = the last step's x_goal."""

    def __init__(self, Q, R, x_goal=None, u_goal=None, Q_final=None, x_goal_final=None):
        self.Q, self.R, self.x_goal, self.u_goal, self.Q_final, self.x_goal_final = Q, R, x_goal, u_goal, Q_final, x_goal_final

    def evaluate(self, X_traj, U):
        """J per environment [B] of X_traj [T+1, B, 2nu] and U [T, B, nu] (None: 0)"""
        X_traj = np.asarray(X_traj, dtype=float)
        T, B, nx = X_traj.shape[0] - 1, X_traj.shape[1], X_traj.shape[2]
        _, _, Q, R, xg, ug, Qf, xgf = cost_arrays(T, B, nx // 2, self.Q, self.R, self.x_goal, self.u_goal, self.Q_final, self.x_goal_final)
        dx = X_traj[:T] - (0.0 if xg is None else xg)
        du = (0.0 if U is None else np.asarray(U, dtype=float)) - (0.0 if ug is None else ug)
        du = np.broadcast_to(du, (T, B, nx // 2))
        # the arrays are column-major per entry: Q[t, e, j, i] = Q_t[i, j]
        J = 0.5 * np.einsum("tbi,tbji,tbj->b", dx, np.broadcast_to(Q, (T, B, nx, nx)), dx)
        J += 0.5 * np.einsum("tbi,tbji,tbj->b", du, np.broadcast_to(R, (T, B) + R.shape[2:]), du)
        dxf = X_traj[T] - (0.0 if xgf is None else xgf)
        return J + 0.5 * np.einsum("bi,bji,bj->b", dxf, np.broadcast_to(Qf, (B, nx, nx)), dxf)


def ilqr(mechanism: Mechanism, x0, U0, cost: QuadraticCost, iterations: int = 20, active=None, opts=None, device: int = 0, mu0: float = 0.0,
         tol: float = 1e-10):
    """iLQR in minimal coordinates for a batch of B problems, as IterativeLQR.jl runs Dojo's examples (trajectory_optimization.md),
    without constraints.  x0 [B, 2nu] or [2nu], U0 [T, nu] or [T, B, nu] the initial inputs, cost a QuadraticCost, active [nu] mask of
    the inputs the optimiser may change (None: all; the others stay at U0).  Every iteration is three device calls:
      1. rollout_minimal_gradients(x0, U): the nominal X and the Jacobians Gx, Gu;
      2. lqr_backward: the gains K, k and the expected decrease dV; where its Cholesky fails, mu is raised for that environment and the
         pass repeated;
      3. a backtracking line search per environment, alpha = 1, 1/2, ..., 1/512: rollout_feedback(K, x_ref = X, u_ref = U + alpha k)
         is accepted when the cost decreases by at least 1e-4 (alpha dV1 + alpha^2 dV2) in magnitude.  The accepted U_applied is the
         next nominal, so the next rollout reproduces the accepted trajectory bit for bit.  Where no trial is accepted, mu is raised and
         the trajectory kept; an environment whose expected decrease falls below tol (1 + J) has converged and keeps its trajectory.
    Returns (X [T+1, B, 2nu], U [T, B, nu], K [T, B, nu, 2nu], k [T, B, nu] (the gains of a final backward pass about X, U), J
    [iterations+1, B] (the cost before each iteration and at the end; non-increasing), status [B]: 0 converged, 1 not converged within
    `iterations`, 2 the backward pass or the line search failed at the largest regularisation (1e8))."""
    x0 = np.asarray(x0, dtype=float)
    X0 = np.atleast_2d(x0)
    B, nu = X0.shape[0], mechanism.nu
    U0 = np.asarray(U0, dtype=float)
    T = U0.shape[0]
    U = np.ascontiguousarray(np.broadcast_to(U0.reshape(T, -1, nu), (T, B, nu)))
    s = _stepper(mechanism, B, device)
    Z0 = s.minimal_to_maximal(X0)
    mu = np.full(B, float(mu0))
    status = np.ones(B, dtype=np.int32)
    hist = []

    def backward(X, U, Gx, Gu):
        K, k, dV, st = s.lqr_backward(X, U, Gx, Gu, cost, mu, active)
        while (st != 0).any() and (mu[st != 0] < 1e8).any():
            mu[st != 0] = np.maximum(10.0 * mu[st != 0], 1e-6)
            K, k, dV, st = s.lqr_backward(X, U, Gx, Gu, cost, mu, active)
        return K, k, dV, st

    X, Gx, Gu, _, _ = s.rollout_minimal_gradients(X0, U, T, opts)
    J = cost.evaluate(X, U)
    for _ in range(iterations):
        hist.append(J)
        K, k, dV, st = backward(X, U, Gx, Gu)
        active_env = (status == 1) & (st == 0)
        status[(status == 1) & (st != 0)] = 2
        converged = active_env & (-(dV[:, 0] + dV[:, 1]) <= tol * (1.0 + np.abs(J)))
        status[converged] = 0
        pending = active_env & ~converged
        if not pending.any():
            break
        K, k = np.nan_to_num(K), np.nan_to_num(k)
        Un = U.copy()
        for alpha in 0.5 ** np.arange(10):
            _, _, traj, Ua, _ = s.rollout_feedback(Z0, T, K, x_ref=X[:T], u_ref=U + alpha * k, opts=opts, record=True)
            Xt = np.stack([X[0]] + [s.maximal_to_minimal(traj[t]) for t in range(T)])
            Jt = cost.evaluate(Xt, Ua)
            ok = pending & np.isfinite(Jt) & (Jt <= J) & (J - Jt >= -1e-4 * (alpha * dV[:, 0] + alpha ** 2 * dV[:, 1]))
            Un[:, ok] = Ua[:, ok]
            pending &= ~ok
            if not pending.any():
                break
        mu[pending] = np.maximum(10.0 * mu[pending], 1e-6)
        status[pending & (mu > 1e8)] = 2
        accepted = active_env & ~converged & ~pending
        mu[accepted] = np.where(mu[accepted] > 1e-6, 0.1 * mu[accepted], mu0)
        U = Un
        X, Gx, Gu, _, _ = s.rollout_minimal_gradients(X0, U, T, opts)
        J = cost.evaluate(X, U)
    while len(hist) < iterations + 1:
        hist.append(J)
    K, k, _, _ = s.lqr_backward(X, U, Gx, Gu, cost, mu, active)
    return X, U, K, k, np.array(hist), status


class Storage:
    """Storage{T,N} (simulation/storage.jl:15-42) for a batch: arrays indexed [step, environment, body, :].
    x, q, v, ω: the state before every solve; px, pq: body momenta (world frame); vl, ωl: velocities derived from them."""

    def __init__(self, traj, sto, diag):
        T, B, _ = traj.shape
        z = traj.reshape(T, B, -1, 13)
        self.x, self.v, self.q, self.ω = z[..., 0:3], z[..., 3:6], z[..., 6:10], z[..., 10:13]
        self.px, self.pq, self.vl, self.ωl = sto[..., 0:3], sto[..., 3:6], sto[..., 6:9], sto[..., 9:12]
        self._diag = diag

    def __len__(self):
        return self.x.shape[0]


def momentum(mechanism: Mechanism, storage: Storage):
    """momentum(mechanism, storage) (mechanics/momentum.jl:1-15): [steps, B, 6] = linear; angular about the centre of mass"""
    return storage._diag[..., 0:6]


def kinetic_energy(mechanism: Mechanism, storage: Storage):
    """kinetic_energy(mechanism, storage) (mechanics/energy.jl:17-41): [steps, B]"""
    return storage._diag[..., 6]


def potential_energy(mechanism: Mechanism, storage: Storage):
    """potential_energy(mechanism, storage) (mechanics/energy.jl:43-93): [steps, B]"""
    return storage._diag[..., 7]


def mechanical_energy(mechanism: Mechanism, storage: Storage):
    """mechanical_energy(mechanism, storage) (mechanics/energy.jl:1-15)"""
    return storage._diag[..., 6] + storage._diag[..., 7]


def simulate_record(mechanism: Mechanism, steps: int, z0=None, control: Optional[Callable] = None, opts=None, device: int = 0) -> Storage:
    """simulate!(mechanism, steps, storage, control!; record=true) -> Storage, everything computed on the device
    (momenta and energies included: save_to_storage!, simulation/storage.jl:50-67)."""
    z0 = mechanism.z0 if z0 is None else z0
    Z = np.atleast_2d(np.asarray(z0, dtype=float))
    B = Z.shape[0]
    if isinstance(control, LinearFeedback):
        raise ValueError("simulate_record: a LinearFeedback controller is not supported (use simulate(..., control=fb, record=True))")
    s = _stepper(mechanism, B, device)
    U = None
    if control is not None:
        U = np.zeros((steps, B, mechanism.nu))
        for k in range(steps):
            uk = control(k)
            if uk is not None:
                U[k] = np.asarray(uk, dtype=float)
    _, traj, sto, diag, _ = s.simulate_record(Z, U, steps, opts)
    return Storage(traj, sto, diag)


def status_name(code: int) -> str:
    return STATUS.get(int(code), "unknown")
