"""Reverse mode through a fused rollout on the H100 (dojo_rollout_tape / dojo_rollout_vjp and dojo_jl_b200.autograd.rollout).

The CPU twin on the kernel emulation is tests/test_rollout_vjp.py; this file checks the device code against dojo_rollout_grad's Jacobians
on the same device, the pointer kinds, the autograd binding and one gradient-descent problem solved with its gradients alone.
"""
import numpy as np
import pytest

import dojo_jl_b200 as dj
from dojo_jl_b200 import capi
from dojo_jl_b200.solver import BatchedStepper
from test_rollout_vjp import TOL, _mech, _start, assert_close, contract

# the legged mechanisms touch down and reach joint limits within T = 12 (see TOL in test_rollout_vjp.py)
GPU_TOL = dict(TOL, quadruped=1e-6, atlas=1e-6)

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _pair(name, B, T, seed, opts=None):
    m = _mech(name)
    s = BatchedStepper(m, B, 0)
    Z0, U = _start(m, B, T, seed)
    return m, s, Z0, U


@pytest.mark.parametrize("name", ("ant", "quadruped", "atlas", "block_linear"))
def test_matches_jacobian_contraction(name):
    B, T = 64, 12
    m, s, Z0, U = _pair(name, B, T, 41)
    traj, Fz, Fu, st, it = s.rollout_grad(Z0, U, T)
    traj2, tape, st2, it2 = s.rollout_tape(Z0, U, T)
    assert np.array_equal(traj, traj2) and np.array_equal(st, st2) and np.array_equal(it, it2)
    gZ = np.random.default_rng(42).normal(size=(T + 1, B, 12 * m.Nb))
    gZ0, gU, vst = s.rollout_vjp(traj2, U, tape, gZ)
    assert (vst == 0).all()
    lam, gUr, lamA, gUa = contract(Fz, Fu, gZ)
    assert_close(gZ0, lam, lamA, f"{name} gZ0", GPU_TOL.get(name, 1e-11))
    assert_close(gU, gUr, gUa, f"{name} gU", GPU_TOL.get(name, 1e-11))
    s.close()


def test_pointer_kinds_are_bit_identical():
    """host pointers, device pointers (synchronous entries) and the _async entries on a torch stream"""
    B, T = 64, 6
    m, s, Z0, U = _pair("ant", B, T, 43)
    traj, tape, st, it = s.rollout_tape(Z0, U, T)
    gZ = np.random.default_rng(44).normal(size=(T + 1, B, 12 * m.Nb))
    gZ0, gU, vst = s.rollout_vjp(traj, U, tape, gZ)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    dZ0, dU, dgZ = d(Z0), d(U), d(gZ)
    for sync in (True, False):
        dtraj, dtape = torch.empty((T + 1, B, m.nz), dtype=torch.float64, device="cuda"), torch.empty((T, B, m.nres), dtype=torch.float64, device="cuda")
        dst, dit = torch.empty((T, B), dtype=torch.int32, device="cuda"), torch.empty((T, B), dtype=torch.int32, device="cuda")
        dgZ0, dgU = torch.empty((B, 12 * m.Nb), dtype=torch.float64, device="cuda"), torch.empty((T, B, m.nu), dtype=torch.float64, device="cuda")
        dvst = torch.empty(B, dtype=torch.int32, device="cuda")
        if sync:
            o = capi.solver_options()
            import ctypes as C
            assert s.L.dojo_rollout_tape(s.h, C.byref(o), B, T, C.c_void_p(dZ0.data_ptr()), C.c_void_p(dU.data_ptr()), C.c_void_p(dtraj.data_ptr()),
                                         C.c_void_p(dtape.data_ptr()), C.c_void_p(dst.data_ptr()), C.c_void_p(dit.data_ptr())) == 0
            assert s.L.dojo_rollout_vjp(s.h, B, T, C.c_void_p(dtraj.data_ptr()), C.c_void_p(dU.data_ptr()), C.c_void_p(dtape.data_ptr()),
                                        C.c_void_p(dgZ.data_ptr()), C.c_void_p(dgZ0.data_ptr()), C.c_void_p(dgU.data_ptr()), C.c_void_p(dvst.data_ptr())) == 0
        else:
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                s.rollout_tape_device(dZ0.data_ptr(), dU.data_ptr(), dtraj.data_ptr(), dtape.data_ptr(), B, T, dstatus=dst.data_ptr(), diters=dit.data_ptr(),
                                      stream=stream.cuda_stream)
                s.rollout_vjp_device(dtraj.data_ptr(), dU.data_ptr(), dtape.data_ptr(), dgZ.data_ptr(), dgZ0.data_ptr(), B, T, dgU=dgU.data_ptr(),
                                     dstatus=dvst.data_ptr(), stream=stream.cuda_stream)
            stream.synchronize()
        for got, ref in ((dtraj, traj), (dtape, tape), (dst, st), (dit, it), (dgZ0, gZ0), (dgU, gU), (dvst, vst)):
            assert np.array_equal(got.cpu().numpy(), ref), sync
    s.close()


def test_tape_matches_rollout():
    B, T = 64, 10
    m, s, Z0, U = _pair("quadruped", B, T, 45)
    traj, tape, st, it = s.rollout_tape(Z0, U, T)
    Zf, st_any, tr = s.rollout(Z0, U, T, record=True)
    assert np.array_equal(traj[1:], tr) and np.array_equal(traj[-1], Zf) and np.array_equal(st.max(axis=0), st_any)
    s.close()


def test_batch_independence():
    """environment e alone equals environment e of the batch, bit for bit"""
    B, T = 8, 5
    m, s, Z0, U = _pair("ant", B, T, 46)
    traj, tape, _, _ = s.rollout_tape(Z0, U, T)
    gZ = np.random.default_rng(47).normal(size=(T + 1, B, 12 * m.Nb))
    ref = s.rollout_vjp(traj, U, tape, gZ)
    for e in (0, 6):
        one = s.rollout_vjp(traj[:, e:e + 1], U[:, e:e + 1], tape[:, e:e + 1], gZ[:, e:e + 1])
        assert np.array_equal(one[0][0], ref[0][e]) and np.array_equal(one[1][:, 0], ref[1][:, e])
    s.close()


def test_autograd_matches_contraction():
    """torch.autograd.grad of a scalar loss through autograd.rollout: the Jacobian contraction after the attitude maps"""
    from dojo_jl_b200.autograd import from_attitude, rollout, to_attitude
    B, T = 16, 8
    m, s, Z0, U = _pair("ant", B, T, 48)
    W = np.random.default_rng(49).normal(size=(T + 1, B, m.nz))
    tZ0 = torch.tensor(Z0, device="cuda", requires_grad=True)
    tU = torch.tensor(U, device="cuda", requires_grad=True)
    Z_traj, status = rollout(m, tZ0, tU)
    loss = (Z_traj * torch.tensor(W, device="cuda")).sum()
    gZ0, gU = torch.autograd.grad(loss, (tZ0, tU))
    traj, Fz, Fu, st, _ = s.rollout_grad(Z0, U, T)
    assert np.array_equal(Z_traj.detach().cpu().numpy(), traj) and np.array_equal(status.cpu().numpy(), st)
    gZ = to_attitude(traj, W)
    lam, gUr, lamA, gUa = contract(Fz, Fu, gZ)
    assert_close(gU.cpu().numpy(), gUr, gUa, "autograd gU", TOL["ant"])
    assert_close(gZ0.cpu().numpy(), from_attitude(Z0, lam), np.abs(from_attitude(Z0, lamA)), "autograd gZ0", TOL["ant"])
    s.close()


def test_autograd_central_differences_pendulum():
    """the pendulum check of the CPU suite, through the autograd path: c' z_T + sum_{t<T} d' z_t at rtol = btol = 1e-11"""
    from dojo_jl_b200.autograd import rollout
    m = _mech("pendulum")
    T = 6
    Z0, U = _start(m, 1, T, seed=29)
    opts = capi.solver_options(rtol=1e-11, btol=1e-11, max_iter=100)
    rng = np.random.default_rng(30)
    c, d = rng.normal(size=m.nz), rng.normal(size=m.nz)
    s = BatchedStepper(m, 1, 0)

    def loss_np(U_):
        Zf, _, tr = s.rollout(Z0, U_, T, opts, record=True)
        return float(c @ Zf[0] + sum(d @ z[0] for z in tr[:-1]) + d @ Z0[0])
    tU = torch.tensor(U, device="cuda", requires_grad=True)
    Z_traj, st = rollout(m, torch.tensor(Z0, device="cuda"), tU, opts)
    tc, td = torch.tensor(c, device="cuda"), torch.tensor(d, device="cuda")
    loss = (Z_traj[T, 0] * tc).sum() + (Z_traj[:T, 0] * td).sum()
    (gU,) = torch.autograd.grad(loss, (tU,))
    eps = 1e-6
    fd = np.zeros_like(U)
    for t in range(T):
        Up, Um = U.copy(), U.copy()
        Up[t, 0, 0] += eps
        Um[t, 0, 0] -= eps
        fd[t, 0, 0] = (loss_np(Up) - loss_np(Um)) / (2 * eps)
    assert np.abs(gU.cpu().numpy() - fd).max() < 1e-6 * max(1.0, np.abs(fd).max())
    s.close()


def pendulum_descent(grad_fn, iters=25):
    """32 pendulums, T = 40 steps of torque, driven to the final position a constant torque of 1.5 reaches: gradient descent on the open-loop
    inputs with a backtracking line search; grad_fn(U) -> (loss [scalar], dloss/dU).  Returns the loss history of the accepted steps."""
    hist = []
    U = np.zeros((40, 32, 1))
    loss, g = grad_fn(U)
    hist.append(loss)
    alpha = 1.0
    for _ in range(iters):
        while alpha > 1e-8:
            Un = U - alpha * g
            ln, gn = grad_fn(Un)
            if ln < loss:
                U, loss, g = Un, ln, gn
                hist.append(loss)
                alpha *= 2.0
                break
            alpha *= 0.5
    return hist


def _pendulum_problem():
    m = _mech("pendulum")
    Z0 = np.tile(m.z0, (32, 1))
    Z0[:, 10:13] += np.random.default_rng(50).normal(0.0, 0.3, (32, 3)) * (m.z0[10:13] != 0 if np.any(m.z0[10:13]) else 1.0)
    return m, Z0


def test_gradient_descent_lowers_the_loss():
    """every accepted step lowers the loss, and after 25 iterations the loss is below 1e-3 of where it started"""
    from dojo_jl_b200.autograd import rollout
    m, Z0 = _pendulum_problem()
    s = BatchedStepper(m, 32, 0)
    target = s.rollout(Z0, np.full((40, 32, 1), 1.5), 40)[0][:, :3]
    tZ0, tt = torch.tensor(Z0, device="cuda"), torch.tensor(target, device="cuda")

    def grad_fn(U):
        tU = torch.tensor(U, device="cuda", requires_grad=True)
        Z_traj, _ = rollout(m, tZ0, tU)
        loss = ((Z_traj[-1, :, :3] - tt) ** 2).sum()
        (g,) = torch.autograd.grad(loss, (tU,))
        return float(loss), g.cpu().numpy()
    hist = pendulum_descent(grad_fn)
    assert all(b < a for a, b in zip(hist, hist[1:]))
    assert hist[-1] < 1e-3 * hist[0], (hist[0], hist[-1])
    s.close()


def test_refusals():
    m = _mech("ant")
    s = BatchedStepper(m, 8, 0)
    import ctypes as C
    T, B = 2, 4
    o = capi.solver_options()
    Z0 = np.tile(m.z0, (B, 1))
    traj, tape = np.empty((T + 1, B, m.nz)), np.empty((T, B, m.nres))
    gZ, gZ0 = np.zeros((T + 1, B, 12 * m.Nb)), np.empty((B, 12 * m.Nb))
    p = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
    L, h = s.L, s.h
    assert L.dojo_rollout_tape(h, C.byref(o), 0, T, p(Z0), None, p(traj), p(tape), None, None) == -1
    assert L.dojo_rollout_tape(h, C.byref(o), 9, T, p(Z0), None, p(traj), p(tape), None, None) == -1
    assert L.dojo_rollout_tape(h, C.byref(o), B, 0, p(Z0), None, p(traj), p(tape), None, None) == -1
    assert L.dojo_rollout_tape(h, C.byref(o), B, T, p(Z0), None, p(traj), None, None, None) == -1
    assert L.dojo_rollout_tape(h, C.byref(o), B, T, p(Z0), None, p(traj), p(tape), None, None) == 0
    assert L.dojo_rollout_vjp(h, B, T, p(traj), None, p(tape), None, p(gZ0), None, None) == -1
    assert L.dojo_rollout_vjp(h, B, T, p(traj), None, p(tape), p(gZ), None, None, None) == -1
    assert L.dojo_rollout_vjp(h, B, 0, p(traj), None, p(tape), p(gZ), p(gZ0), None, None) == -1
    assert L.dojo_rollout_vjp(h, 9, T, p(traj), None, p(tape), p(gZ), p(gZ0), None, None) == -1
    assert L.dojo_rollout_vjp_async(h, B, T, None, None, None, None, None, None, None, None) == -1
    assert L.dojo_rollout_vjp(h, B, T, p(traj), None, p(tape), p(gZ), p(gZ0), None, None) == 0
    assert np.array_equal(gZ0, np.zeros_like(gZ0))
    s.close()
