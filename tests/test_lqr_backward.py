"""Riccati backward pass of iLQR / TVLQR (dojo_lqr_backward) -- CPU suite on the kernel emulation.

dojo_lqr_backward_kernel (dojo.jl_b200/csrc/dojo_lqr.cuh) runs here on the CPU fibers of tests/hostemu/cuda_shim.h (tests/hostemu/lqr.py)
and is compared with the recursion written out in numpy below, for the (2nu, nu) of every bundled mechanism; with explicitly tiled cost
arrays; with an active-input mask; with the stationary gain of scipy's discrete algebraic Riccati equation; with a failing Cholesky and
its regularisation; and under every thread order of the emulation.  The -m gpu twin is tests/test_zzzzzzzz_gpu_lqr.py.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (2nu, nu) of pendulum, cartpole, block, quadruped, raiberthopper-sized, ant, humanoid-sized and atlas
SIZES = ((2, 1), (4, 2), (12, 6), (14, 7), (28, 14), (36, 18), (72, 36))


class Cost:
    def __init__(self, Q, R, x_goal=None, u_goal=None, Q_final=None, x_goal_final=None):
        self.Q, self.R, self.x_goal, self.u_goal, self.Q_final, self.x_goal_final = Q, R, x_goal, u_goal, Q_final, x_goal_final


def _emu(nu):
    from hostemu.lqr import LqrEmu
    return LqrEmu(nu)


def _threads(nu):
    """the CTA size dojo_lqr_backward launches with (lqr_threads in dojo_b200.cu)"""
    return 64 if nu <= 4 else 128 if nu <= 16 else 256 if nu <= 24 else 512


def _spd(rng, n, lead=()):
    G = rng.normal(size=lead + (n, n))
    return G @ np.swapaxes(G, -1, -2) / n + 0.5 * np.eye(n)


def _problem(nu, B, T, seed):
    """random nominal trajectory, Jacobians with spectral radius near 1, SPD per-(step, environment) costs and random goals"""
    rng = np.random.default_rng(seed)
    nx = 2 * nu
    O, _ = np.linalg.qr(rng.normal(size=(T, B, nx, nx)))
    A = O * rng.uniform(0.95, 1.02, (T, B, 1, nx)) + 0.02 * rng.normal(size=(T, B, nx, nx))
    Bu = 0.3 * rng.normal(size=(T, B, nx, nu))
    X = rng.normal(size=(T + 1, B, nx))
    U = rng.normal(size=(T, B, nu))
    cost = Cost(_spd(rng, nx, (T, B)), _spd(rng, nu, (T, B)), rng.normal(size=(T, B, nx)), rng.normal(size=(T, B, nu)), _spd(rng, nx, (B,)),
                rng.normal(size=(B, nx)))
    return X, U, A, Bu, cost


def _full(cost, T, B, nu, nx=None):
    """the cost arrays broadcast to explicit per-(step, environment) arrays, row-major matrices (a reduced problem, nx != 2 nu, must
    give them so already)"""
    from dojo_jl_b200.solver import cost_arrays
    if nx is not None and nx != 2 * nu:
        return cost.Q, cost.R, cost.x_goal, cost.u_goal, cost.Q_final, cost.x_goal_final
    steps, envs, Q, R, xg, ug, Qf, xgf = cost_arrays(T, B, nu, cost.Q, cost.R, cost.x_goal, cost.u_goal, cost.Q_final, cost.x_goal_final)
    nx = 2 * nu
    tile = lambda a, tail: np.broadcast_to(a, (T, B) + tail) if a is not None else np.zeros((T, B) + tail)
    Qf = np.broadcast_to(Qf.swapaxes(1, 2), (B, nx, nx))
    xgf = np.zeros((B, nx)) if xgf is None else np.broadcast_to(xgf, (B, nx))
    return tile(Q.swapaxes(2, 3), (nx, nx)), tile(R.swapaxes(2, 3), (nu, nu)), tile(xg, (nx,)), tile(ug, (nu,)), Qf, xgf


def riccati(X, U, A, Bu, cost, mu=None, active=None):
    """the recursion of dojo_lqr.cuh in plain numpy, one environment at a time; Quu factored on the active inputs only"""
    T, B, nx, nu = A.shape[0], A.shape[1], A.shape[2], Bu.shape[3]
    Q, R, xg, ug, Qf, xgf = _full(cost, T, B, nu, nx)
    U = np.zeros((T, B, nu)) if U is None else U
    act = np.arange(nu) if active is None else np.flatnonzero(np.asarray(active))
    K, k = np.zeros((T, B, nu, nx)), np.zeros((T, B, nu))
    dV, status = np.zeros((B, 2)), np.zeros(B, dtype=np.int32)
    for e in range(B):
        m = 0.0 if mu is None else np.broadcast_to(mu, (B,))[e]
        P = Qf[e].copy()
        p = Qf[e] @ (X[T, e] - xgf[e])
        for t in range(T - 1, -1, -1):
            At, Bt = A[t, e], Bu[t, e][:, act]
            Qx = Q[t, e] @ (X[t, e] - xg[t, e]) + At.T @ p
            Qu = (R[t, e] @ (U[t, e] - ug[t, e]))[act] + Bt.T @ p
            Qxx = Q[t, e] + At.T @ P @ At
            Quu = R[t, e][np.ix_(act, act)] + Bt.T @ P @ Bt
            Qux = Bt.T @ P @ At
            try:
                Lc = np.linalg.cholesky(Quu + m * np.eye(len(act)))
            except np.linalg.LinAlgError:
                status[e] = t + 1
                K[: t + 1, e] = np.nan
                k[: t + 1, e] = np.nan
                dV[e] = np.nan
                break
            Ka = np.linalg.solve(Lc.T, np.linalg.solve(Lc, Qux))
            ka = -np.linalg.solve(Lc.T, np.linalg.solve(Lc, Qu))
            K[t, e][act], k[t, e][act] = Ka, ka
            P = Qxx + Ka.T @ Quu @ Ka - Ka.T @ Qux - Qux.T @ Ka
            P = 0.5 * (P + P.T)
            p = Qx - Ka.T @ Quu @ ka - Ka.T @ Qu + Qux.T @ ka
            dV[e] += [ka @ Qu, 0.5 * ka @ Quu @ ka]
    return K, k, dV, status


def _close(got, ref, tol, what):
    for name, g, r in zip(("K", "k", "dV"), got[:3], ref[:3]):
        scale = max(1.0, float(np.abs(r).max()))
        err = float(np.abs(g - r).max()) / scale
        assert err < tol, (what, name, err)


@pytest.mark.parametrize("nx,nu", SIZES)
def test_against_numpy(nx, nu):
    """K, k and dV of the kernel == the numpy recursion to 1e-10 relative, for every mechanism size; the CTA size changes nothing"""
    B, T = 2, 3
    X, U, A, Bu, cost = _problem(nu, B, T, seed=nu)
    emu = _emu(nu)
    got = emu.backward(X, U, A, Bu, cost, threads=_threads(nu))
    ref = riccati(X, U, A, Bu, cost)
    assert (got[3] == 0).all()
    _close(got, ref, 1e-10, (nx, nu))
    for threads in (32, 96):  # every output element is one thread's fixed-order sum, whichever thread
        other = emu.backward(X, U, A, Bu, cost, threads=threads)
        for g, o in zip(got, other):
            assert np.array_equal(g, o), threads


def test_smem_bytes():
    """the shared-memory working set: atlas fits the H100's 227 KB opt-in maximum per block"""
    assert _emu(36).smem_bytes() == 202624 <= 227 * 1024
    assert _emu(38).smem_bytes() <= 227 * 1024 < _emu(39).smem_bytes()


def test_broadcast_equals_tiled():
    """shared, per-step, per-environment and per-(step, environment) cost arrays == the same arrays tiled explicitly, bit for bit"""
    nu, B, T = 3, 3, 4
    nx = 2 * nu
    rng = np.random.default_rng(5)
    X, U, A, Bu, _ = _problem(nu, B, T, seed=6)
    emu = _emu(nu)
    cases = [Cost(_spd(rng, nx), _spd(rng, nu)),
             Cost(_spd(rng, nx), _spd(rng, nu), rng.normal(size=nx), rng.normal(size=nu), _spd(rng, nx), rng.normal(size=nx)),
             Cost(_spd(rng, nx, (B,)), _spd(rng, nu), rng.normal(size=(B, nx)), None, _spd(rng, nx, (B,))),
             Cost(_spd(rng, nx, (T, 1)), _spd(rng, nu, (T, B)), rng.normal(size=(T, 1, nx)), rng.normal(size=(T, B, nu))),
             Cost(_spd(rng, nx), _spd(rng, nu), x_goal_final=rng.normal(size=(B, nx)))]
    for i, c in enumerate(cases):
        Q, R, xg, ug, Qf, xgf = _full(c, T, B, nu)
        tiled = Cost(np.array(Q), np.array(R), np.array(xg), np.array(ug), np.array(Qf), np.array(xgf))
        got, ref = emu.backward(X, U, A, Bu, c), emu.backward(X, U, A, Bu, tiled)
        for g, r in zip(got, ref):
            assert np.array_equal(g, r), i
    # the defaults: Q_final = the last step's Q, x_goal_final = the last step's x_goal
    c = cases[3]
    explicit = Cost(c.Q, c.R, c.x_goal, c.u_goal, np.broadcast_to(c.Q[-1, 0], (nx, nx)), c.x_goal[-1, 0])
    for g, r in zip(emu.backward(X, U, A, Bu, c), emu.backward(X, U, A, Bu, explicit)):
        assert np.array_equal(g, r)


def test_cost_arrays_refuse_bad_shapes():
    from dojo_jl_b200.solver import cost_arrays
    nu, B, T = 2, 3, 4
    Q, R = np.eye(4), np.eye(2)
    for bad in (dict(Q=np.eye(3)), dict(R=np.ones((B + 1, nu, nu))), dict(Q_final=np.ones((T, B, 4, 4))), dict(x_goal=np.ones((T + 1, 1, 4)))):
        args = dict(Q=Q, R=R)
        args.update(bad)
        with pytest.raises(ValueError):
            cost_arrays(T, B, nu, **args)


def test_active_mask():
    """inactive rows of K and entries of k are exactly 0; the active part == the numpy recursion on the reduced problem
    (B[:, act], R[act, act], u and u_goal restricted to the active inputs)"""
    nu, B, T = 7, 3, 5
    X, U, A, Bu, cost = _problem(nu, B, T, seed=9)
    active = np.array([0, 1, 1, 0, 1, 0, 1], dtype=np.int32)
    act = np.flatnonzero(active)
    U[..., active == 0] = 0.0
    cost.u_goal[..., active == 0] = 0.0
    K, k, dV, st = _emu(nu).backward(X, U, A, Bu, cost, active=active, threads=_threads(nu))
    assert (st == 0).all()
    assert (K[:, :, active == 0] == 0).all() and (k[:, :, active == 0] == 0).all()
    red = Cost(cost.Q, cost.R[..., act[:, None], act], cost.x_goal, cost.u_goal[..., act], cost.Q_final, cost.x_goal_final)
    Kr, kr, dVr, _ = riccati(X, U[..., act], A, Bu[..., act], red)
    _close((K[:, :, act], k[..., act], dV), (Kr, kr, dVr), 1e-10, "active")
    # the masked recursion with full R rows (the kernel's definition) for a U that is not zero on the inactive inputs
    X, U, A, Bu, cost = _problem(nu, B, T, seed=10)
    _close(_emu(nu).backward(X, U, A, Bu, cost, active=active), riccati(X, U, A, Bu, cost, active=active), 1e-10, "active, full rows")


def _dare_case():
    import scipy.linalg as sl
    rng = np.random.default_rng(3)
    nu, nx = 2, 4
    A = np.eye(nx) + 0.01 * rng.normal(size=(nx, nx))
    A[:2, 2:] += 0.01 * np.eye(2)
    Bm = 0.01 * rng.normal(size=(nx, nu)) + np.vstack([np.zeros((2, 2)), 0.01 * np.eye(2)])
    Q, R = np.eye(nx), np.diag([1.0, 2.0])
    P = sl.solve_discrete_are(A, Bm, Q, R)
    Kd = np.linalg.solve(R + Bm.T @ P @ Bm, Bm.T @ P @ A)
    return nu, A, Bm, Q, R, P, Kd


def test_stationary_lqr_equals_dare():
    """constant A, B with Q_final = the DARE solution: every K_t == the DARE gain to 1e-9; with Q_final = Q and a long horizon, K_0
    converges to it"""
    nu, A, Bm, Q, R, P, Kd = _dare_case()
    B, T = 2, 30
    X, U = np.zeros((T + 1, B, 2 * nu)), np.zeros((T, B, nu))
    As, Bs = np.broadcast_to(A, (T, B) + A.shape), np.broadcast_to(Bm, (T, B) + Bm.shape)
    K, k, dV, st = _emu(nu).backward(X, U, As, Bs, Cost(Q, R, Q_final=P))
    assert (st == 0).all() and (k == 0).all()
    assert np.abs(K - Kd).max() / np.abs(Kd).max() < 1e-9
    T = 3000
    X, U = np.zeros((T + 1, 1, 2 * nu)), np.zeros((T, 1, nu))
    As, Bs = np.broadcast_to(A, (T, 1) + A.shape), np.broadcast_to(Bm, (T, 1) + Bm.shape)
    K, _, _, _ = _emu(nu).backward(X, U, As, Bs, Cost(Q, R))
    assert np.abs(K[0, 0] - Kd).max() / np.abs(Kd).max() < 1e-9
    assert np.abs(K[-1, 0] - Kd).max() / np.abs(Kd).max() > 1e-3  # the horizon's end is far from stationary


def test_failure_and_regularisation():
    """an indefinite R in one environment: its status is the failing step + 1, its K / k up to that step and its dV are NaN, the other
    environments equal a run without it bit for bit, and a large enough mu for it clears the failure"""
    nu, B, T = 3, 4, 5
    X, U, A, Bu, cost = _problem(nu, B, T, seed=12)
    emu = _emu(nu)
    clean = emu.backward(X, U, A, Bu, cost)
    assert (clean[3] == 0).all()
    bad = Cost(cost.Q, cost.R.copy(), cost.x_goal, cost.u_goal, cost.Q_final, cost.x_goal_final)
    bad.R[2, 1] = -50.0 * np.eye(nu)  # Quu is indefinite at step 2 only
    K, k, dV, st = emu.backward(X, U, A, Bu, bad)
    assert st.tolist() == [0, 3, 0, 0]
    assert np.isnan(K[:3, 1]).all() and np.isnan(k[:3, 1]).all() and np.isnan(dV[1]).all()
    assert np.array_equal(K[3:, 1], clean[0][3:, 1]) and np.array_equal(k[3:, 1], clean[1][3:, 1])
    others = [0, 2, 3]
    for g, r in zip((K, k), clean[:2]):
        assert np.array_equal(g[:, others], r[:, others])
    assert np.array_equal(dV[others], clean[2][others]) and np.array_equal(st[others], clean[3][others])
    ref = riccati(X, U, A, Bu, bad)
    assert ref[3].tolist() == st.tolist()
    mu = np.array([0.0, 200.0, 0.0, 0.0])
    K2, k2, dV2, st2 = emu.backward(X, U, A, Bu, bad, mu=mu)
    assert (st2 == 0).all()
    _close((K2, k2, dV2), riccati(X, U, A, Bu, bad, mu=mu), 1e-10, "mu")
    assert np.array_equal(K2[:, 0], clean[0][:, 0])


ORDERS = r"""
import sys, numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests")
from test_lqr_backward import _emu, _problem, _threads
out = {}
for nu in (2, 14, 36):
    X, U, A, Bu, cost = _problem(nu, 2, 3, seed=40 + nu)
    for k, v in enumerate(_emu(nu).backward(X, U, A, Bu, cost, mu=np.array([0.0, 1e-3]), active=np.arange(nu) %% 5 != 1, threads=_threads(nu))):
        out[f"{nu}_{k}"] = v
np.savez(sys.argv[1], **out)
"""


def _run_order(order, path):
    env = dict(os.environ)
    env.pop("HOSTEMU_ORDER", None)
    if order:
        env["HOSTEMU_ORDER"] = order
    r = subprocess.run([sys.executable, "-c", ORDERS % {"root": ROOT}, path], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    if order:
        assert "thread order of a round = " + order in r.stderr
    return np.load(path)


def test_thread_orders_are_bit_identical(tmp_path):
    """HOSTEMU_ORDER=reverse|random: a missing barrier between the phases of a step would show here"""
    ref = _run_order(None, str(tmp_path / "asc.npz"))
    for order in ("reverse", "random"):
        got = _run_order(order, str(tmp_path / (order + ".npz")))
        for k in ref.files:
            assert np.array_equal(ref[k], got[k], equal_nan=True), (order, k)


def test_ctypes_mirror_matches_the_c_header(tmp_path):
    """DojoQuadraticCost: size and field offsets as the C compiler lays them out == the ctypes mirror in dojo.jl_b200/capi.py"""
    from dojo_jl_b200 import capi
    st = capi.DojoQuadraticCost
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "dojo_b200.h")}"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(DojoQuadraticCost));']
    lines += [f'  printf("{f} %zu\\n", offsetof(DojoQuadraticCost, {f}));' for f, _ in st._fields_]
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-o", str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(out["size"]) == C.sizeof(st)
    for f, _ in st._fields_:
        assert int(out[f]) == getattr(st, f).offset, f


def test_quadratic_cost_evaluate():
    """QuadraticCost.evaluate == an explicit loop over steps and environments"""
    from dojo_jl_b200.api import QuadraticCost
    nu, B, T = 3, 4, 5
    X, U, _, _, c = _problem(nu, B, T, seed=21)
    rng = np.random.default_rng(22)
    for cost in (QuadraticCost(c.Q, c.R, c.x_goal, c.u_goal, c.Q_final, c.x_goal_final),
                 QuadraticCost(c.Q[:, :1], c.R[0, 0], None, c.u_goal[0, 0]),
                 QuadraticCost(_spd(rng, 2 * nu, (B,)), c.R[:, :1], c.x_goal[0], x_goal_final=rng.normal(size=2 * nu))):
        Q, R, xg, ug, Qf, xgf = _full(cost, T, B, nu)
        ref = np.zeros(B)
        for e in range(B):
            for t in range(T):
                dx, du = X[t, e] - xg[t, e], U[t, e] - ug[t, e]
                ref[e] += 0.5 * dx @ Q[t, e] @ dx + 0.5 * du @ R[t, e] @ du
            dx = X[T, e] - xgf[e]
            ref[e] += 0.5 * dx @ Qf[e] @ dx
        got = cost.evaluate(X, U)
        assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
