"""Reverse mode in minimal coordinates on the H100: dojo_maximal_to_minimal_vjp / dojo_minimal_to_maximal_vjp, their composition with the
rollout tape and adjoint (api.get_minimal_trajectory_vjp, autograd.rollout_minimal) and a closed loop started from a minimal state.

The reference is the dense maximal recursion on the same device: dojo_rollout_grad's Fz / Fu, dojo_maximal_to_minimal_jacobian at every
slab and dojo_minimal_to_maximal_jacobian at z_0.  The CPU twin is tests/test_minimal_vjp.py.
"""
import ctypes as C

import numpy as np
import pytest

import dojo_jl_b200 as dj
from dojo_jl_b200 import api, capi
from dojo_jl_b200.solver import BatchedStepper
from test_rollout_vjp import _mech, _start, contract

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

EINVAL = -1  # DOJO_EINVAL of include/dojo_b200.h
GPU_TOL = {"ant": 1e-6, "quadruped": 1e-6, "atlas": 1e-6, "block_linear": 1e-10}


def _rel_close(got, ref, bound, what, tol):
    """|got - ref| <= tol * (bound + max of bound over the vector): test_rollout_vjp.assert_close"""
    scale = bound + bound.max(axis=-1, keepdims=True)
    err = np.abs(got - ref)
    ok = err <= tol * np.maximum(scale, 1e-300)
    assert np.isfinite(got).all() and ok.all(), f"{what}: worst {np.max(err / np.maximum(scale, 1e-300)):.2e} at {np.argwhere(~ok)[:4].tolist()}"


def _moving_states(m, s, B, seed):
    """B maximal states on the map's manifold with nonzero joint velocities: minimal_to_maximal of a started state plus velocity noise"""
    Z0, _ = _start(m, B, 1, seed)
    X = s.maximal_to_minimal(Z0)
    rng = np.random.default_rng(seed + 1)
    off = 0
    for j in m.joints:
        n = j.input_dimension
        X[:, 2 * off + n:2 * off + 2 * n] += rng.normal(0.0, 0.5, (B, n))
        off += n
    return s.minimal_to_maximal(X)


# ----------------------------------------------------------------------------------------------------- the two map adjoints
@pytest.mark.parametrize("name", ("ant", "quadruped", "atlas", "block_linear"))
def test_map_adjoints_match_dense_jacobians(name):
    """M(z)' gX and N(z)' gZ against the dense map Jacobians of the same device, contracted; and n = B (T+1) > max_batch states in one call"""
    m = _mech(name)
    B = 64
    s = BatchedStepper(m, B, 0)
    Z = _moving_states(m, s, B, 301)
    rng = np.random.default_rng(302)
    gX, gZ = rng.normal(size=(B, 2 * m.nu)), rng.normal(size=(B, 12 * m.Nb))
    M, N = s.maximal_to_minimal_jacobian(Z), s.minimal_to_maximal_jacobian(Z)
    gotM, gotN = s.maximal_to_minimal_vjp(Z, gX), s.minimal_to_maximal_vjp(Z, gZ)
    _rel_close(gotM, np.einsum("bij,bi->bj", M, gX), np.einsum("bij,bi->bj", np.abs(M), np.abs(gX)), f"{name} M'", 1e-12)
    _rel_close(gotN, np.einsum("bij,bi->bj", N, gZ), np.einsum("bij,bi->bj", np.abs(N), np.abs(gZ)), f"{name} N'", 1e-12)
    # a whole trajectory's slabs in one call: n = 13 B > max_batch; each state's result equals the one of the batch above
    T = 12
    Zt = np.concatenate([Z] * (T + 1))
    gXt, gZt = np.concatenate([gX] * (T + 1)), np.concatenate([gZ] * (T + 1))
    bigM, bigN = s.maximal_to_minimal_vjp(Zt, gXt), s.minimal_to_maximal_vjp(Zt, gZt)
    assert Zt.shape[0] > s.max_batch
    assert np.array_equal(bigM, np.concatenate([gotM] * (T + 1))) and np.array_equal(bigN, np.concatenate([gotN] * (T + 1)))
    s.close()


def test_pointer_kinds_and_batch_independence_are_bit_identical():
    """host pointers, device pointers through the synchronous entries and the _async entries on a torch stream give the same bits; state
    e alone equals state e among 64"""
    m = dj.get_mechanism("atlas")
    B = 64
    s = BatchedStepper(m, B, 0)
    Z = _moving_states(m, s, B, 311)
    rng = np.random.default_rng(312)
    gX, gZ = rng.normal(size=(B, 2 * m.nu)), rng.normal(size=(B, 12 * m.Nb))
    refM, refN = s.maximal_to_minimal_vjp(Z, gX), s.minimal_to_maximal_vjp(Z, gZ)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    dZ, dgX, dgZ = dev(Z), dev(gX), dev(gZ)
    for kind in ("sync", "async"):
        oM = torch.full((B, 12 * m.Nb), -1.0, dtype=torch.float64, device="cuda")
        oN = torch.full((B, 2 * m.nu), -1.0, dtype=torch.float64, device="cuda")
        if kind == "sync":
            assert s.L.dojo_maximal_to_minimal_vjp(s.h, B, C.c_void_p(dZ.data_ptr()), C.c_void_p(dgX.data_ptr()), C.c_void_p(oM.data_ptr())) == 0
            assert s.L.dojo_minimal_to_maximal_vjp(s.h, B, C.c_void_p(dZ.data_ptr()), C.c_void_p(dgZ.data_ptr()), C.c_void_p(oN.data_ptr())) == 0
        else:
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                s.maximal_to_minimal_vjp_device(dZ.data_ptr(), dgX.data_ptr(), oM.data_ptr(), B, stream=stream.cuda_stream)
                s.minimal_to_maximal_vjp_device(dZ.data_ptr(), dgZ.data_ptr(), oN.data_ptr(), B, stream=stream.cuda_stream)
            stream.synchronize()
        assert np.array_equal(oM.cpu().numpy(), refM) and np.array_equal(oN.cpu().numpy(), refN), kind
    for e in (0, 37):
        assert np.array_equal(s.maximal_to_minimal_vjp(Z[e:e + 1], gX[e:e + 1])[0], refM[e])
        assert np.array_equal(s.minimal_to_maximal_vjp(Z[e:e + 1], gZ[e:e + 1])[0], refN[e])
    s.close()


def test_refusals_launch_nothing():
    """n <= 0, null buffers and a null handle return DOJO_EINVAL before any launch"""
    m = dj.get_mechanism("ant")
    s = BatchedStepper(m, 4, 0)
    Z = np.tile(m.z0, (4, 1))
    gX, gZ, out = np.zeros((4, 2 * m.nu)), np.zeros((4, 12 * m.Nb)), np.zeros((4, 12 * m.Nb))
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
    n0 = s.launch_count
    for name in ("dojo_maximal_to_minimal_vjp", "dojo_minimal_to_maximal_vjp"):
        f = getattr(s.L, name)
        fa = getattr(s.L, name + "_async")
        assert f(s.h, 0, p(Z), p(gX), p(out)) == EINVAL and f(s.h, -3, p(Z), p(gX), p(out)) == EINVAL
        for args in ((None, gX, out), (Z, None, out), (Z, gX, None)):
            assert f(s.h, 4, *[p(a) for a in args]) == EINVAL
            assert fa(s.h, 4, *[p(a) for a in args], None) == EINVAL
        assert f(None, 4, p(Z), p(gX), p(out)) == EINVAL
    assert s.launch_count == n0
    s.close()


# ----------------------------------------------------------------------------------------------------- the rollout composition
def dense_reference(s, m, X0, U, gX):
    """the dense maximal recursion on the device's Jacobians: (gX0, gU, bounds)"""
    T, B = U.shape[0], U.shape[1]
    traj, Fz, Fu, st, _ = s.rollout_grad(s.minimal_to_maximal(X0), U, T)
    M = np.stack([s.maximal_to_minimal_jacobian(traj[t]) for t in range(T + 1)])
    gZ = np.einsum("tbij,tbi->tbj", M, gX)
    gZa = np.einsum("tbij,tbi->tbj", np.abs(M), np.abs(gX))
    lam, gUr, _, _ = contract(Fz, Fu, gZ)
    _, _, lamA, gUa = contract(np.abs(Fz), np.abs(Fu), gZa)
    N0 = s.minimal_to_maximal_jacobian(traj[0])
    return np.einsum("bij,bi->bj", N0, lam), gUr, np.einsum("bij,bi->bj", np.abs(N0), lamA), gUa, traj, st


@pytest.mark.parametrize("name", ("ant", "quadruped", "atlas", "block_linear"))
def test_rollout_minimal_matches_dense_recursion(name):
    """autograd.rollout_minimal: X_traj equals dojo_rollout_minimal_gradients' bit for bit; X0.grad / U.grad against the dense recursion"""
    from dojo_jl_b200 import autograd
    m = _mech(name)
    B, T = 64, 12
    s = BatchedStepper(m, B, 0)
    Z0, U = _start(m, B, T, 321)
    X0 = s.maximal_to_minimal(Z0)
    gX = np.random.default_rng(322).normal(size=(T + 1, B, 2 * m.nu))
    tX0 = torch.tensor(X0, device="cuda", requires_grad=True)
    tU = torch.tensor(U, device="cuda", requires_grad=True)
    Xt, status = autograd.rollout_minimal(m, tX0, tU)
    (Xt * torch.tensor(gX, device="cuda")).sum().backward()
    Xr, _, _, str_, _ = s.rollout_minimal_gradients(X0, U, T)
    assert np.array_equal(Xt.detach().cpu().numpy(), Xr) and np.array_equal(status.cpu().numpy(), str_)
    gX0r, gUr, gX0a, gUa, _, _ = dense_reference(s, m, X0, U, gX)
    _rel_close(tX0.grad.cpu().numpy(), gX0r, gX0a, f"{name} X0.grad", GPU_TOL[name])
    _rel_close(tU.grad.cpu().numpy(), gUr, gUa, f"{name} U.grad", GPU_TOL[name])
    s.close()


@pytest.mark.parametrize("name", ("ant", "block_linear"))
def test_get_minimal_trajectory_vjp_matches_dense_recursion(name):
    """api.get_minimal_trajectory_vjp, batched and single-environment, against the same recursion"""
    m = _mech(name)
    B, T = 16, 8
    s = BatchedStepper(m, B, 0)
    Z0, U = _start(m, B, T, 331)
    X0 = s.maximal_to_minimal(Z0)
    gX = np.random.default_rng(332).normal(size=(T + 1, B, 2 * m.nu))
    Xt, gX0, gU, st = api.get_minimal_trajectory_vjp(m, X0, U, gX)
    gX0r, gUr, gX0a, gUa, traj, str_ = dense_reference(s, m, X0, U, gX)
    assert Xt.shape == (T + 1, B, 2 * m.nu) and np.array_equal(st, str_)
    assert np.array_equal(Xt, np.stack([s.maximal_to_minimal(traj[t]) for t in range(T + 1)]))
    _rel_close(gX0, gX0r, gX0a, f"{name} gX0", GPU_TOL[name])
    _rel_close(gU, gUr, gUa, f"{name} gU", GPU_TOL[name])
    x1, g1, u1, s1 = api.get_minimal_trajectory_vjp(m, X0[3], U[:, 3], gX[:, 3])
    assert x1.shape == (T + 1, 2 * m.nu) and g1.shape == (2 * m.nu,) and u1.shape == (T, m.nu) and s1.shape == (T,)
    assert np.array_equal(x1, Xt[:, 3]) and np.array_equal(g1, gX0[3]) and np.array_equal(u1, gU[:, 3])
    s.close()


def _minimal_loss(m, X0, U, d, opts):
    from dojo_jl_b200 import autograd
    Xt, st = autograd.rollout_minimal(m, X0, U, opts)
    assert (st == 0).all()
    return (Xt * d).sum()


@pytest.mark.parametrize("name", ("pendulum", "cartpole"))
def test_rollout_minimal_central_differences(name):
    """sum_t d_t' x_t at rtol = btol = 1e-11: X0.grad and U.grad against central differences (1e-6 relative)"""
    m = _mech(name)
    T = 6
    s = BatchedStepper(m, 1, 0)
    Z0, U = _start(m, 1, T, 341)
    X0 = torch.tensor(s.maximal_to_minimal(Z0), device="cuda", requires_grad=True)
    tU = torch.tensor(U, device="cuda", requires_grad=True)
    d = torch.tensor(np.random.default_rng(342).normal(size=(T + 1, 1, 2 * m.nu)), device="cuda")
    opts = capi.solver_options(rtol=1e-11, btol=1e-11, max_iter=100)
    _minimal_loss(m, X0, tU, d, opts).backward()
    eps = 1e-6
    with torch.no_grad():
        fd_x = torch.zeros_like(X0)
        for k in range(2 * m.nu):
            e = torch.zeros_like(X0)
            e[0, k] = eps
            fd_x[0, k] = (_minimal_loss(m, X0 + e, tU, d, opts) - _minimal_loss(m, X0 - e, tU, d, opts)) / (2 * eps)
        fd_u = torch.zeros_like(tU)
        for t in range(T):
            for j in range(m.nu):
                e = torch.zeros_like(tU)
                e[t, 0, j] = eps
                fd_u[t, 0, j] = (_minimal_loss(m, X0, tU + e, d, opts) - _minimal_loss(m, X0, tU - e, d, opts)) / (2 * eps)
    scale = max(1.0, fd_x.abs().max().item(), fd_u.abs().max().item())
    assert (X0.grad - fd_x).abs().max().item() < 1e-6 * scale
    assert (tU.grad - fd_u).abs().max().item() < 1e-6 * scale
    s.close()


def test_closed_loop_from_a_minimal_start_central_differences():
    """autograd.rollout_feedback started from autograd.minimal_to_maximal(X0), a PID pendulum: X0.grad against central differences"""
    from dojo_jl_b200 import autograd
    m = dj.get_mechanism("pendulum")
    T, nx = 20, 2
    f64 = dict(dtype=torch.float64, device="cuda")
    K = torch.tensor([[8.0, 1.5]], **f64)
    K_i = torch.tensor([[2.0, 0.0]], **f64)
    x_ref = torch.tensor([0.6, 0.0], **f64)
    d = torch.tensor(np.random.default_rng(351).normal(size=(T + 1, 1, nx)), **f64)
    opts = capi.solver_options(rtol=1e-11, btol=1e-11, max_iter=100)

    def loss(X0):
        _, Xt, _ = autograd.rollout_feedback(m, autograd.minimal_to_maximal(m, X0), K, x_ref=x_ref, K_i=K_i, opts=opts, T=T)
        return (Xt * d).sum()

    X0 = torch.tensor([[0.3, -0.4]], requires_grad=True, **f64)
    loss(X0).backward()
    eps = 1e-6
    with torch.no_grad():
        fd = torch.zeros_like(X0)
        for k in range(nx):
            e = torch.zeros_like(X0)
            e[0, k] = eps
            fd[0, k] = (loss(X0 + e) - loss(X0 - e)) / (2 * eps)
    scale = max(1.0, fd.abs().max().item())
    assert (X0.grad - fd).abs().max().item() < 1e-6 * scale, (X0.grad, fd)
