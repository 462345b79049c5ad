"""Riccati backward pass and iLQR on the H100 (run with -m gpu): dojo_lqr_backward on the Jacobians of real rollouts agrees with the numpy
recursion; host pointers, device pointers and the async entry agree bit for bit; cartpole_lqr.jl's gain comes out of the device; the
iLQR driver swings a pendulum batch up and pushes a block to its goal; refused calls launch nothing.  The CPU twin is
tests/test_lqr_backward.py."""
import ctypes as C

import numpy as np
import pytest

import dojo_jl_b200 as dj
from conftest import jittered_states
from dojo_jl_b200 import api, capi
from test_lqr_backward import Cost, _close, _spd, riccati

pytestmark = pytest.mark.gpu

DOJO_EINVAL = -1
B, T = 64, 12


def _mech(name):
    if name == "block_linear":
        return dj.get_mechanism("block", contact_type="linear")
    return dj.get_mechanism(name)


def _unactuated(m):
    """the active mask of the actuated inputs: a floating base (a joint without impulses) is inactive"""
    act = np.ones(m.nu, dtype=np.int32)
    off = 0
    for j in m.joints:
        if j.nimpulses == 0:
            act[off:off + j.input_dimension] = 0
        off += j.input_dimension
    return act


def _nominal(st, m, seed):
    """X_traj, U, Gx, Gu of a real rollout from jittered states under small random inputs"""
    rng = np.random.default_rng(seed)
    if m.name == "block":
        Z = np.tile(m.z0, (B, 1))
        Z[:, 2] += rng.uniform(-0.9, 0.0, B)
    else:
        Z = jittered_states(m, B, rng)
    X0 = st.maximal_to_minimal(Z)
    U = rng.normal(0.0, 0.2, (T, B, m.nu)) * _unactuated(m)
    X, Gx, Gu, status, _ = st.rollout_minimal_gradients(X0, U, T)
    return X, U, Gx, Gu


def _cost(m, seed):
    rng = np.random.default_rng(seed)
    nx = 2 * m.nu
    return Cost(_spd(rng, nx, (B,)), np.eye(m.nu) * 0.1, rng.normal(0.0, 0.1, (T, B, nx)), None, 10.0 * np.eye(nx))


@pytest.mark.parametrize("name", ("ant", "quadruped", "atlas", "block_linear"))
def test_real_jacobians_against_numpy(name):
    """the device recursion on real Jacobians == numpy to 1e-9 relative (the floating base inactive where there is one)"""
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech(name)
    st = BatchedStepper(m, B)
    X, U, Gx, Gu = _nominal(st, m, seed=51)
    cost = _cost(m, seed=52)
    active = None if m.name == "block" else _unactuated(m)
    mu = np.full(B, 1e-6)
    got = st.lqr_backward(X, U, Gx, Gu, cost, mu=mu, active=active)
    ref = riccati(X, U, Gx, Gu, cost, mu=mu, active=active)
    assert (got[3] == ref[3]).all()
    ok = got[3] == 0
    assert ok.any()
    _close((got[0][:, ok], got[1][:, ok], got[2][ok]), (ref[0][:, ok], ref[1][:, ok], ref[2][ok]), 1e-9, name)
    if active is not None:
        assert (got[0][:, :, active == 0] == 0).all() and (got[1][:, :, active == 0] == 0).all()
    st.close()


def test_pointer_kinds_agree():
    """host pointers, device pointers and dojo_lqr_backward_async on a torch stream: bit-identical outputs"""
    import torch
    from dojo_jl_b200.solver import BatchedStepper, cost_arrays
    m = _mech("ant")
    st = BatchedStepper(m, B)
    X, U, Gx, Gu = _nominal(st, m, seed=53)
    cost = _cost(m, seed=54)
    active, mu = _unactuated(m), np.linspace(0.0, 1e-3, B)
    ref = st.lqr_backward(X, U, Gx, Gu, cost, mu=mu, active=active)
    nu, nx = m.nu, 2 * m.nu
    steps, envs, Q, R, xg, ug, Qf, xgf = cost_arrays(T, B, nu, cost.Q, cost.R, cost.x_goal, cost.u_goal, cost.Q_final, cost.x_goal_final)
    dev = lambda a: None if a is None else torch.from_numpy(np.array(a)).cuda()
    d = {k: dev(v) for k, v in dict(X=X, U=U, Gx=np.swapaxes(Gx, 2, 3), Gu=np.swapaxes(Gu, 2, 3), Q=Q, R=R, xg=xg, ug=ug, Qf=Qf, xgf=xgf,
                                      mu=mu).items()}
    p = lambda t: None if t is None else t.data_ptr()
    for kind in ("sync", "async"):
        K = torch.empty((T, B, nx, nu), dtype=torch.float64, device="cuda")
        k = torch.empty((T, B, nu), dtype=torch.float64, device="cuda")
        dV = torch.empty((B, 2), dtype=torch.float64, device="cuda")
        status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        if kind == "sync":
            c = capi.DojoQuadraticCost(steps, envs, *[None if d.get(n) is None else C.cast(C.c_void_p(d[n].data_ptr()), capi.c_double_p)
                                                      for n in ("Q", "R", "xg", "ug", "Qf", "xgf")])
            act = np.ascontiguousarray(active, dtype=np.int32)
            rc = st.L.dojo_lqr_backward(st.h, B, T, C.byref(c), C.c_void_p(act.ctypes.data), *[C.c_void_p(p(t)) if t is not None else None for t in
                                        (d["X"], d["U"], d["Gx"], d["Gu"], d["mu"], K, k, dV, status)])
            assert rc == 0, st.L.dojo_last_error(st.h)
        else:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                st.lqr_backward_device(B, T, p(d["X"]), p(d["Gx"]), p(d["Gu"]), p(K), p(k), p(d["Q"]), p(d["R"]), p(d["Qf"]), steps=steps, envs=envs,
                                       dx_goal=p(d["xg"]), dx_goal_final=p(d["xgf"]), dU=p(d["U"]), dmu=p(d["mu"]), active=active, ddV=p(dV), dstatus=p(status),
                                       stream=s.cuda_stream)
            s.synchronize()
        got = (K.cpu().numpy().swapaxes(2, 3), k.cpu().numpy(), dV.cpu().numpy(), status.cpu().numpy())
        for g, r in zip(got, ref):
            assert np.array_equal(g, r), kind
    st.close()


def test_cartpole_lqr_gain_on_the_device():
    """cartpole_lqr.jl: linearised at 0, the cart input active only, Q = I, R = 1, Q_final = the DARE solution: every K_t == the gain
    test_cartpole_lqr_batch computes with scipy to 1e-9, and rollout_feedback under it stabilises the batch as that test does"""
    import scipy.linalg as sl
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech("cartpole")
    A, Bu = api.get_minimal_gradients(m, np.zeros(2 * m.nu), np.zeros(m.nu))
    B1 = Bu[:, :1]
    P = sl.solve_discrete_are(A, B1, np.eye(2 * m.nu), np.eye(1))
    Kref = np.zeros((m.nu, 2 * m.nu))
    Kref[0] = np.linalg.solve(np.eye(1) + B1.T @ P @ B1, B1.T @ P @ A)[0]
    st = BatchedStepper(m, B)
    Tn = 50
    X = np.zeros((Tn + 1, B, 2 * m.nu))
    Gx, Gu = np.broadcast_to(A, (Tn, B) + A.shape), np.broadcast_to(Bu, (Tn, B) + Bu.shape)
    K, k, dV, status = st.lqr_backward(X, None, Gx, Gu, Cost(np.eye(2 * m.nu), np.eye(m.nu), Q_final=P), active=[1, 0])
    assert (status == 0).all() and (k == 0).all() and (dV == 0).all()
    assert np.abs(K - Kref).max() / np.abs(Kref).max() < 1e-9
    X0 = np.zeros((B, 2 * m.nu))
    X0[:, 2] = np.linspace(-0.3, 0.3, B)
    steps = int(round(20.0 / m.timestep))
    Zf, s_any, _, Ua, _ = st.rollout_feedback(st.minimal_to_maximal(X0), steps, K[0])
    assert (s_any == 0).all() and (Ua[:, :, 1] == 0).all()
    xf = np.abs(st.maximal_to_minimal(Zf)).max(axis=1)
    assert (xf < 1e-3).all(), xf.max()
    st.close()


def _check_history(J):
    assert np.isfinite(J).all()
    assert (np.diff(J, axis=0) <= 0).all(), np.diff(J, axis=0).max()


def test_ilqr_pendulum_swing_up():
    """pendulum swing-up (trajectory_optimization.md): 32 initial angles hanging near the bottom, goal upright (theta = pi), torque cost;
    every environment ends within 1e-2 rad of upright with |theta_dot| < 1e-2, the cost history never increases, and dojo_rollout
    driven by the final U reproduces the final X bit for bit"""
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech("pendulum")
    Bn, Tn = 32, 100
    x0 = np.zeros((Bn, 2))
    x0[:, 0] = np.linspace(-0.5, 0.5, Bn)
    goal = np.array([np.pi, 0.0])
    cost = api.QuadraticCost(np.diag([1e-2, 1e-2]), 1e-3 * np.eye(1), x_goal=goal, Q_final=1e4 * np.eye(2))
    X, U, K, k, J, status = api.ilqr(m, x0, np.zeros((Tn, 1)), cost, iterations=60)
    _check_history(J)
    err = np.abs(X[-1] - goal)
    print("pendulum: final |theta - pi| max %.2e, |theta_dot| max %.2e, status %s, J %s" % (err[:, 0].max(), err[:, 1].max(), np.bincount(status),
                                                                                          J[-1].max()))
    assert (err[:, 0] < 1e-2).all() and (err[:, 1] < 1e-2).all()
    st = BatchedStepper(m, Bn)
    Z0 = st.minimal_to_maximal(x0)
    _, _, traj = st.rollout(Z0, U, Tn, record=True)
    Xr = np.stack([st.maximal_to_minimal(traj[t]) for t in range(Tn)])
    assert np.array_equal(Xr, X[1:])
    assert K.shape == (Tn, Bn, 1, 2) and k.shape == (Tn, Bn, 1)
    st.close()


def test_ilqr_block_to_goal():
    """a block pushed to a goal 1 m along x by forces on its centre of mass (torques inactive), from rest on the ground with linear
    contact: it ends within 5 cm of the goal and the cost history never increases"""
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech("block_linear")
    Bn, Tn = 4, 100
    st = BatchedStepper(m, Bn)
    Zrest, _ = st.rollout(np.tile(m.z0, (Bn, 1)), None, 200)  # settle on the ground
    x0 = st.maximal_to_minimal(Zrest)
    x0[:, 6:] = 0.0
    goal = x0[0].copy()
    goal[0] += 1.0
    active = np.array([1, 1, 1, 0, 0, 0], dtype=np.int32)
    Q = np.diag([1.0] * 3 + [0.1] * 3 + [0.1] * 6)
    cost = api.QuadraticCost(1e-2 * Q, 1e-3 * np.eye(6), x_goal=goal, Q_final=1e2 * Q)
    X, U, K, k, J, status = api.ilqr(m, x0, np.zeros((Tn, 6)), cost, iterations=40, active=active)
    _check_history(J)
    err = np.linalg.norm(X[-1, :, :3] - goal[:3], axis=1)
    print("block: final position error max %.3e m, status %s" % (err.max(), np.bincount(status)))
    assert (err < 0.05).all(), err
    assert (U[..., 3:] == 0).all()
    st.close()


def test_refusals():
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech("ant")
    st = BatchedStepper(m, 8)
    nu, nx = m.nu, 2 * m.nu
    Tn, Bn = 2, 4
    big = np.zeros(nx * nx * 9 * 3)  # enough entries for every array of these calls
    bp = capi.dptr(big)
    out = np.empty(nx * nx * 9 * 3)
    op = capi.dptr(out)
    L = st.L
    n = st.launch_count
    none_active = np.zeros(nu, dtype=np.int32)

    def call(Bn=Bn, Tn=Tn, c="ok", active=None, X=bp, Gx=bp, Gu=bp, K=op, k=op):
        cost = {"ok": C.byref(capi.DojoQuadraticCost(1, 1, bp, bp, None, None, bp, None)), None: None}.get(c, c)
        a = None if active is None else C.c_void_p(active.ctypes.data)
        return L.dojo_lqr_backward(st.h, Bn, Tn, cost, a, X, None, Gx, Gu, None, K, k, None, None)

    cc = lambda steps=1, envs=1, Q=bp, R=bp, Qf=bp: C.byref(capi.DojoQuadraticCost(steps, envs, Q, R, None, None, Qf, None))
    refused = [call(Bn=9), call(Bn=0), call(Tn=0), call(c=None), call(c=cc(Q=None)), call(c=cc(R=None)), call(c=cc(Qf=None)),
               call(X=None), call(Gx=None), call(Gu=None), call(K=None), call(k=None), call(c=cc(steps=3)), call(c=cc(envs=2)),
               call(active=none_active)]
    refused.append(L.dojo_lqr_backward_async(st.h, 9, Tn, cc(), None, bp, None, bp, bp, None, op, op, None, None, None))
    assert refused == [DOJO_EINVAL] * len(refused), refused
    assert st.launch_count == n
    assert call(c=cc(steps=Tn, envs=Bn)) == 0 and st.launch_count == n + 1
    st.close()
