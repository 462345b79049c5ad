"""Closed-loop rollouts on the H100 (run with -m gpu): dojo_rollout driven by the returned U_applied reproduces dojo_rollout_feedback's
trajectory bit for bit, and so does dojo_rollout_grad; the host- and device-pointer entries agree; the reference's control examples run
batched (cartpole LQR, pendulum PID); refused calls launch nothing.  The CPU twin is tests/test_rollout_feedback.py."""
import ctypes as C

import numpy as np
import pytest

import dojo_jl_b200 as dj
from conftest import jittered_states
from dojo_jl_b200 import api, capi

pytestmark = pytest.mark.gpu

DOJO_EINVAL = -1
B, T = 64, 12


def _mech(name):
    if name == "block_linear":
        return dj.get_mechanism("block", contact_type="linear")
    return dj.get_mechanism(name)


def _start(m, B, seed):
    rng = np.random.default_rng(seed)
    if m.name == "block":
        Z = np.tile(m.z0, (B, 1))
        Z[:, 2] += rng.uniform(-0.9, 0.0, B)
        Z[:, 3:6] = rng.normal(size=(B, 3)) * [1.0, 1.0, 0.3]
        Z[:, 10:13] = rng.normal(size=(B, 3))
    elif m.Nb > 2:
        Z = jittered_states(m, B, rng)
    else:
        Z = np.tile(m.z0, (B, 1)) + rng.normal(0.0, 1e-3, (B, m.nz)) * (np.arange(m.nz) % 13 >= 10)
    return Z


def _law(m, B, T, seed, scale=0.3):
    rng = np.random.default_rng(seed)
    nu = m.nu
    return dict(K=rng.normal(0.0, scale, (T, B, nu, 2 * nu)), K_i=rng.normal(0.0, scale, (T, B, nu, 2 * nu)),
                x_ref=rng.normal(0.0, 0.1, (T, B, 2 * nu)), u_ref=rng.normal(0.0, 0.3, (T, B, nu)), xi=rng.normal(0.0, 0.05, (B, 2 * nu)))


def _same(got, ref, what):
    for k, (g, r) in enumerate(zip(got, ref)):
        assert g.shape == r.shape, (what, k, g.shape, r.shape)
        assert np.array_equal(g, r, equal_nan=True), f"{what}: output {k} differs (max |diff| {np.nanmax(np.abs(g - r))})"


@pytest.mark.parametrize("name", ("ant", "quadruped", "atlas", "block_linear"))
def test_equals_open_loop_rollout(name):
    """dojo_rollout and dojo_rollout_grad driven by U_applied reproduce the closed loop bit for bit (the forward kernel dojo_rollout
    picks may be the small-mechanism one; the FB kernel is generic)"""
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech(name)
    st = BatchedStepper(m, B)
    Z0 = _start(m, B, seed=41)
    Zf, s_any, traj, Ua, xi = st.rollout_feedback(Z0, T, **_law(m, B, T, seed=42), record=True)
    assert np.isfinite(Ua).all() and np.isfinite(xi).all()
    Zo, so, trajo = st.rollout(Z0, Ua, T, record=True)
    _same((traj, Zf, s_any), (trajo, Zo, so), name)
    trajg, _, _, sg, _ = st.rollout_grad(Z0, Ua, T)
    assert np.array_equal(trajg[1:], traj) and np.array_equal(sg.max(axis=0), s_any)
    st.close()


def test_host_and_device_pointers_agree():
    import torch
    from dojo_jl_b200.solver import BatchedStepper, feedback_arrays
    m = _mech("ant")
    st = BatchedStepper(m, B)
    Z0 = _start(m, B, seed=43)
    law = _law(m, B, T, seed=44)
    host = st.rollout_feedback(Z0, T, **law, record=True)
    steps, envs, K, xr, ur, Ki = feedback_arrays(T, B, m.nu, law["K"], law["x_ref"], law["u_ref"], law["K_i"])
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dZ0, dK, dKi, dxr, dur, dxi = cu(Z0), cu(K), cu(Ki), cu(xr), cu(ur), cu(law["xi"])
    dZf = torch.empty_like(dZ0)
    dtraj = torch.empty((T, B, st.nz), dtype=torch.float64, device="cuda")
    dUa = torch.empty((T, B, st.nu), dtype=torch.float64, device="cuda")
    dst = torch.empty(B, dtype=torch.int32, device="cuda")
    st.rollout_feedback_device(dZ0.data_ptr(), dZf.data_ptr(), B, T, dK.data_ptr(), steps, envs, dK_i=dKi.data_ptr(), dx_ref=dxr.data_ptr(),
                               du_ref=dur.data_ptr(), dxi=dxi.data_ptr(), dtraj=dtraj.data_ptr(), dU_applied=dUa.data_ptr(), dstatus=dst.data_ptr(),
                               stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    dev = (dZf.cpu().numpy(), dst.cpu().numpy(), dtraj.cpu().numpy(), dUa.cpu().numpy(), dxi.cpu().numpy())
    _same(dev, host, "device vs host")
    # device pointers through the host-or-device entry, without U_applied and Z_traj
    dxi.copy_(cu(law["xi"]))
    fb = capi.DojoFeedback(steps, envs, C.cast(C.c_void_p(dK.data_ptr()), capi.c_double_p), C.cast(C.c_void_p(dKi.data_ptr()), capi.c_double_p),
                           C.cast(C.c_void_p(dxr.data_ptr()), capi.c_double_p), C.cast(C.c_void_p(dur.data_ptr()), capi.c_double_p))
    dZf.zero_()
    rc = st.L.dojo_rollout_feedback(st.h, None, B, T, dZ0.data_ptr(), C.byref(fb), dxi.data_ptr(), dZf.data_ptr(), None, None, None)
    assert rc == 0
    assert np.array_equal(dZf.cpu().numpy(), host[0]) and np.array_equal(dxi.cpu().numpy(), host[4])
    st.close()


def test_cartpole_lqr_batch():
    """cartpole_lqr.jl batched: an LQR on the cart input from the linearisation at x = 0 (Q = I, R = 1) stabilises every pole angle in
    [-0.3, 0.3] to |x|_inf < 1e-3 within 20 s (the slow cart mode of this LQR is what takes the time)"""
    import scipy.linalg as sl
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech("cartpole")
    A, Bu = api.get_minimal_gradients(m, np.zeros(2 * m.nu), np.zeros(m.nu))
    B1 = Bu[:, :1]
    P = sl.solve_discrete_are(A, B1, np.eye(2 * m.nu), np.eye(1))
    K = np.zeros((m.nu, 2 * m.nu))
    K[0] = np.linalg.solve(np.eye(1) + B1.T @ P @ B1, B1.T @ P @ A)[0]
    st = BatchedStepper(m, B)
    X0 = np.zeros((B, 2 * m.nu))
    X0[:, 2] = np.linspace(-0.3, 0.3, B)
    steps = int(round(20.0 / m.timestep))
    Zf, s_any, _, Ua, _ = st.rollout_feedback(st.minimal_to_maximal(X0), steps, K)
    assert (s_any == 0).all()
    assert (Ua[:, :, 1] == 0).all()
    xf = np.abs(st.maximal_to_minimal(Zf)).max(axis=1)
    assert (xf < 1e-3).all(), xf.max()
    # the api form: one environment, the same law
    fb = api.LinearFeedback(K)
    zf = api.simulate(m, steps, st.minimal_to_maximal(X0[-1:])[0], control=fb)
    assert np.array_equal(zf, Zf[-1])
    st.close()


def test_pendulum_pid_sweep():
    """pendulum_pid.jl with a gain sweep across the batch: environment 0 runs the example's gains and agrees with a host loop of oracle
    steps under the same law to 1e-8 over all 500 steps, ending within 1e-3 rad of the goal; every environment equals its own B = 1 run"""
    from oracle.oracle import Oracle
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech("pendulum")
    rng = np.random.default_rng(45)
    g = np.column_stack([rng.uniform(15, 35, B), rng.uniform(3, 7, B), rng.uniform(30, 70, B)])  # Kp, Kd, Ki
    g[0] = (25.0, 5.0, 50.0)
    K = g[:, None, :2].copy()
    Ki = np.zeros((B, 1, 2))
    Ki[:, 0, 0] = g[:, 2]
    goal = np.array([np.pi / 2, 0.0])
    o = Oracle(m)
    z0 = o.minimal_to_maximal(np.zeros(2))
    st = BatchedStepper(m, B)
    Zf, s_any, traj, Ua, xi = st.rollout_feedback(np.tile(z0, (B, 1)), 500, K, x_ref=goal, K_i=Ki, record=True)
    assert (s_any == 0).all()
    z, s, ref = z0, 0.0, []
    for k in range(500):
        x = o.maximal_to_minimal(z)
        s += (goal[0] - x[0]) * m.timestep
        u = 25.0 * (goal[0] - x[0]) + 50.0 * s + 5.0 * (0.0 - x[1])
        r = o.step(z, np.array([u]))
        z = r[0] if isinstance(r, tuple) else r
        ref.append(z)
    err = np.abs(traj[:, 0] - np.array(ref)).max()
    assert err < 1e-8, err
    assert abs(o.maximal_to_minimal(Zf[0])[0] - goal[0]) < 1e-3
    for e in (0, 1, B - 1):
        one = st.rollout_feedback(z0[None], 500, K[e], x_ref=goal, K_i=Ki[e], record=True)
        assert np.array_equal(one[2][:, 0], traj[:, e]) and np.array_equal(one[4][0], xi[e]), e
    # api: a second call continues the integral, as the example's global summed_error does
    fb = api.LinearFeedback(K[0], x_ref=goal, K_i=Ki[0])
    zh = api.simulate(m, 250, z0, control=fb)
    zf = api.simulate(m, 250, zh, control=fb)
    assert np.array_equal(zf, Zf[0]) and np.array_equal(fb.xi, xi[0])
    with pytest.raises(ValueError):
        api.simulate(m, 10, z0, control=fb, opts=capi.solver_options(verbose=True))
    st.close()


def _welded():
    """one body welded to the world: no inputs"""
    from dojo_jl_b200.mechanism import Body, Joint, Mechanism
    from test_translational_joints import _element
    m = Mechanism("welded", [Body("b", 1.0, np.diag([0.1, 0.1, 0.1]))], [Joint("weld", -1, 0, _element(3), _element(3))], [], timestep=0.01,
                  gravity=(0.0, 0.0, -9.81))
    m.z0 = m.forward_kinematics({})
    return m


def test_refusals():
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech("ant")
    st = BatchedStepper(m, 8)
    Z = _start(m, 9, seed=46)
    nu = m.nu
    K = np.zeros((2, 4, 2 * nu, nu))  # enough entries for steps = T = 2, envs = B = 4
    Kp = capi.dptr(K)
    xi = np.zeros((9, 2 * nu))
    Zf, Ua = np.empty_like(Z), np.empty((2, 9, nu))
    n = st.launch_count
    L = st.L

    def call(Bn, Tn, fb, xip=xi):
        return L.dojo_rollout_feedback(st.h, None, Bn, Tn, capi.dptr(Z), fb, None if xip is None else capi.dptr(xip), capi.dptr(Zf), None, capi.dptr(Ua), None)

    fb = lambda steps=1, envs=1, k=Kp, ki=None: C.byref(capi.DojoFeedback(steps, envs, k, ki, None, None))
    refused = [call(9, 2, fb()), call(0, 2, fb()), call(4, 0, fb()), call(4, 2, None), call(4, 2, fb(k=None)), call(4, 2, fb(steps=3)),
               call(4, 2, fb(envs=2)), call(4, 2, fb(ki=Kp), xip=None)]
    for Bn in (9, 0):  # the async entry refuses the same way
        refused.append(L.dojo_rollout_feedback_async(st.h, None, Bn, 2, None, fb(), None, None, None, None, None, None))
    assert refused == [DOJO_EINVAL] * len(refused), refused
    assert st.launch_count == n
    assert call(4, 2, fb(steps=2, envs=4)) == 0  # steps = T, envs = B
    st.close()
    w = BatchedStepper(_welded(), 4)
    assert w.nu == 0
    n = w.launch_count
    Zw = np.tile(w.mech.z0, (2, 1))
    one = np.zeros(1)
    rc = w.L.dojo_rollout_feedback(w.h, None, 2, 2, capi.dptr(Zw), C.byref(capi.DojoFeedback(1, 1, capi.dptr(one), None, None, None)), None,
                                   capi.dptr(np.empty_like(Zw)), None, None, None)
    assert rc == DOJO_EINVAL and w.launch_count == n
    w.close()
