"""Reverse mode through a closed-loop rollout (dojo_rollout_feedback_tape + dojo_rollout_feedback_vjp) -- CPU suite on the kernel emulation.

The tape is dojo_rollout_feedback recorded like dojo_rollout_tape, so its trajectory, inputs, integral state, status and iterations must
equal both bit for bit.  The adjoint is checked against the closed-loop recursion built in numpy from rollout_grad's Jacobians at the
applied inputs and the dense maximal-to-minimal Jacobians, against central differences of the closed loop, and for independence of the
slot count, the plan placement, the thread order and the batch.  The -m gpu twin is tests/test_zzzzzzzzzzzz_gpu_feedback_vjp.py.
"""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import dojo_jl_b200 as dj
from conftest import jittered_states
from dojo_jl_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ("pendulum", "cartpole", "ant", "quadruped", "raiberthopper", "block_linear")
TOL = {"ant": 1e-6}  # the accuracy floor of the transposed solve on ant's contact and limit rows (tests/test_rollout_vjp.py)


def _mech(name):
    if name == "block_linear":
        return dj.get_mechanism("block", contact_type="linear")
    return dj.get_mechanism(name)


def _emu(m):
    from hostemu.feedback_vjp import FeedbackVjpEmu
    return FeedbackVjpEmu(m)


def _slots_grad(m):
    return 1 if m.Nb > 13 else 2


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
        Z = np.tile(m.z0, (B, 1)) + rng.normal(0.0, 1e-1, (B, m.nz)) * (np.arange(m.nz) % 13 >= 10)
    return Z


def _law(m, T, B, seed, integral=False, tiled=True):
    """a stabilising-ish time-varying law: small random gains per (step, environment), references near the start"""
    rng = np.random.default_rng(seed)
    nu, nx = m.nu, 2 * m.nu
    sh = (T, B) if tiled else ()
    law = dict(K=rng.normal(0.0, 0.3, sh + (nu, nx)), x_ref=rng.normal(0.0, 0.1, sh + (nx,)), u_ref=rng.normal(0.0, 0.3, sh + (nu,)))
    if integral:
        law["K_i"] = rng.normal(0.0, 0.3, sh + (nu, nx))
    return law


def _full(a, T, B, tail):
    a = np.asarray(a, dtype=np.float64)
    if a.shape == tail:
        a = a[None, None]
    elif a.ndim == len(tail) + 1:
        a = a[None]
    return np.broadcast_to(a, (T, B) + tail)


def dense_recursion(m, rec, law, gZ, gX, gUa, jac, mjac):
    """the closed-loop adjoint recursion in numpy, from the step Jacobians jac(Z0, U, T) -> (Fz, Fu) [T, B, 12Nb, .] at the applied inputs
    and the dense M(z_t) = mjac(Z) [B, 2nu, 12Nb] -- and the same recursion in absolute values (the bound of assert_close)"""
    T, B = rec["tape"].shape[:2]
    nu, nx, h = m.nu, 2 * m.nu, m.timestep
    Fz, Fu = jac(rec["Z_traj"][0], rec["U"], T)
    M = np.stack([mjac(rec["Z_traj"][t]) for t in range(T + 1)])
    K = _full(law["K"], T, B, (nu, nx))
    Ki = _full(law["K_i"], T, B, (nu, nx)) if "K_i" in law else None
    xr = _full(law.get("x_ref", np.zeros(nx)), T, B, (nx,))
    mv = lambda A, v: np.einsum("bij,bi->bj", A, v)  # noqa: E731  (A' v per environment)
    lam = gZ[T] + mv(M[T], gX[T])
    lamA = np.abs(gZ[T]) + mv(np.abs(M[T]), np.abs(gX[T]))
    nv, nvA = np.zeros((B, nx)), np.zeros((B, nx))
    out = {k: np.zeros((T,) + s) for k, s in (("K", (B, nu, nx)), ("K_i", (B, nu, nx)), ("x_ref", (B, nx)), ("u_ref", (B, nu)))}
    bnd = {k: np.zeros_like(v) for k, v in out.items()}
    for t in range(T - 1, -1, -1):
        a = mv(Fu[t], lam) + gUa[t]
        aA = mv(np.abs(Fu[t]), lamA) + np.abs(gUa[t])
        if Ki is not None:
            nv, nvA = nv - np.einsum("bik,bi->bk", Ki[t], a), nvA + np.einsum("bik,bi->bk", np.abs(Ki[t]), aA)
        db = -np.einsum("bik,bi->bk", K[t], a) + h * nv
        dbA = np.einsum("bik,bi->bk", np.abs(K[t]), aA) + h * nvA
        d = rec["X_traj"][t] - xr[t]
        out["u_ref"][t], bnd["u_ref"][t] = a, aA
        out["x_ref"][t], bnd["x_ref"][t] = -db, dbA
        out["K"][t], bnd["K"][t] = -a[:, :, None] * d[:, None, :], aA[:, :, None] * np.abs(d)[:, None, :]
        if Ki is not None:
            xi = rec["Xi_traj"][t]
            out["K_i"][t], bnd["K_i"][t] = -a[:, :, None] * xi[:, None, :], aA[:, :, None] * np.abs(xi)[:, None, :]
        lam = mv(Fz[t], lam) + gZ[t] + mv(M[t], db + gX[t])
        lamA = mv(np.abs(Fz[t]), lamA) + np.abs(gZ[t]) + mv(np.abs(M[t]), dbA + np.abs(gX[t]))
    return dict(gZ0=lam, gxi0=nv, **out), dict(gZ0=lamA, gxi0=nvA, **bnd)


def assert_close(got, ref, bound, what, tol):
    """|got - ref| <= tol * (bound + the bound's largest entry in the same vector), as tests/test_rollout_vjp.py"""
    got, ref, bound = (np.asarray(x).reshape(x.shape[:2] + (-1,)) if np.ndim(x) > 2 else np.asarray(x) for x in (got, ref, bound))
    scale = bound + bound.max(axis=-1, keepdims=True)
    err = np.abs(got - ref)
    ok = err <= tol * scale
    assert ok.all(), f"{what}: worst {np.max(err / np.maximum(scale, 1e-300)):.2e} of the bound at {np.argwhere(~ok)[:4].tolist()}"


def _cotangents(m, T, B, seed):
    rng = np.random.default_rng(seed)
    return (rng.normal(size=(T + 1, B, 12 * m.Nb)), rng.normal(size=(T + 1, B, 2 * m.nu)), rng.normal(size=(T, B, m.nu)))


# ----------------------------------------------------------------------------------------------------- M' w
def test_max_to_min_vjp_matches_dense_jacobian():
    """max_to_min_vjp_joint + the per-body fold against J' w of the dense maximal_to_minimal_jacobian, every mechanism and all 16 joint
    prototypes (tests/hostcheck)"""
    from hostcheck.kinjac_vjp import KinJacVjp, mechanisms
    rng = np.random.default_rng(31)
    for name, m in mechanisms():
        hc = KinJacVjp(m)
        Z = jittered_states(m, 3, rng) if m.Nb > 1 else np.tile(m.z0, (3, 1)) + rng.normal(0.0, 0.2, (3, m.nz)) * (np.arange(m.nz) % 13 >= 3)
        W = rng.normal(size=(3, 2 * m.nu))
        J = hc.maximal_to_minimal_jacobian(Z)
        ref = np.einsum("bij,bi->bj", J, W)
        got = hc.max_to_min_vjp(Z, W)
        scale = np.einsum("bij,bi->bj", np.abs(J), np.abs(W)).max(axis=1, keepdims=True)
        assert np.all(np.abs(got - ref) <= 1e-13 * np.maximum(scale, 1e-300)), (name, np.max(np.abs(got - ref) / np.maximum(scale, 1e-300)))


# ----------------------------------------------------------------------------------------------------- the tape
@pytest.mark.parametrize("integral", (False, True))
@pytest.mark.parametrize("name", CASES)
def test_tape_matches_rollouts(name, integral):
    """Z_traj / U_applied / final xi / status / iterations equal dojo_rollout_feedback's; Z_traj / tape / status / iterations equal
    rollout_tape(Z0, U_applied)'s; X_traj / Xi_traj are the law's x_t / xi_t"""
    m = _mech(name)
    em = _emu(m)
    B, T = 3, 5
    Z0 = _start(m, B, 41)
    law = _law(m, T, B, 42, integral)
    rec = em.rollout_feedback_tape(Z0, T, **law)
    Zf, st_any, traj, Ua, xi, x_last = em.rollout_feedback(Z0, T, **law)
    assert np.array_equal(rec["Z_traj"][1:], traj) and np.array_equal(rec["Z_traj"][-1], Zf) and np.array_equal(rec["U"], Ua)
    assert np.array_equal(rec["status"].max(axis=0), st_any) and np.array_equal(rec["X_traj"][T - 1], x_last)
    if integral:
        assert np.array_equal(rec["xi"], xi) and np.array_equal(rec["Xi_traj"][-1], xi)
    traj2, tape2, st2, it2 = em.rollout_tape(Z0, rec["U"], T, slots=2, grid=2)
    assert np.array_equal(rec["Z_traj"], traj2) and np.array_equal(rec["tape"], tape2)
    assert np.array_equal(rec["status"], st2) and np.array_equal(rec["iters"], it2)
    assert np.isfinite(rec["X_traj"]).all()


# ----------------------------------------------------------------------------------------------------- the adjoint
def test_open_loop_reduction():
    """K = 0, no K_i, no gX / gUa: gZ0 and du_ref are rollout_vjp's gZ0 and gU, bit for bit"""
    m = _mech("cartpole")
    em = _emu(m)
    B, T = 3, 6
    Z0 = _start(m, B, 43)
    law = dict(K=np.zeros((m.nu, 2 * m.nu)), u_ref=np.random.default_rng(44).normal(0.0, 0.5, (T, B, m.nu)))
    rec = em.rollout_feedback_tape(Z0, T, **law)
    gZ = _cotangents(m, T, B, 45)[0]
    got = em.rollout_feedback_vjp(rec, **law, gZ=gZ, slots_grad=2, grid=2)
    gZ0, gU, st = em.rollout_vjp(rec["Z_traj"], rec["U"], rec["tape"], gZ, slots_grad=2, grid=2)
    assert (got["status"] == 0).all() and (st == 0).all()
    assert np.array_equal(got["gZ0"], gZ0) and np.array_equal(got["u_ref"], gU)


@pytest.mark.parametrize("integral", (False, True))
@pytest.mark.parametrize("name", CASES)
def test_matches_dense_recursion(name, integral):
    """every output against the numpy recursion on rollout_grad's Jacobians and the dense M(z_t), random cotangents on every slab"""
    m = _mech(name)
    em = _emu(m)
    B, T = 3, 6 if m.Nb > 2 else 10
    Z0 = _start(m, B, 51)
    law = _law(m, T, B, 52, integral)
    rec = em.rollout_feedback_tape(Z0, T, **law)
    gZ, gX, gUa = _cotangents(m, T, B, 53)
    got = em.rollout_feedback_vjp(rec, **law, gZ=gZ, gX=gX, gUa=gUa, slots_grad=_slots_grad(m), grid=2)
    assert (got["status"] == 0).all(), got["status"]
    ref, bnd = dense_recursion(m, rec, law, gZ, gX, gUa, lambda Z0, U, T: em.rollout_grad(Z0, U, T, slots=2, slots_grad=_slots_grad(m), grid=2)[1:3],
                               lambda Z: em.kinjac(0, Z))
    tol = TOL.get(name, 1e-10)
    keys = ["gZ0", "K", "x_ref", "u_ref"] + (["K_i", "gxi0"] if integral else [])
    for k in keys:
        assert_close(got[k], ref[k], bnd[k], f"{name} {k}", tol)


def test_pendulum_pid_central_differences():
    """dL / d(Kp, Ki, Kd, xi0, x_ref) of a PID pendulum against central differences, solver tolerances 1e-11"""
    m = _mech("pendulum")
    em = _emu(m)
    B, T = 2, 30
    opts = capi.solver_options(rtol=1e-11, btol=1e-11)
    Z0 = _start(m, B, 61)
    rng = np.random.default_rng(62)
    p = dict(kp=rng.uniform(5, 10, B), ki=rng.uniform(0.5, 2, B), kd=rng.uniform(0.5, 2, B), xi0=rng.normal(0, 0.1, (B, 2)),
             xr=rng.normal(0, 0.1, (B, 2)))
    target = 0.3

    def loss_of(q):
        law = dict(K=np.stack([q["kp"], q["kd"]], -1)[:, None, :], K_i=np.stack([q["ki"], np.zeros(B)], -1)[:, None, :], x_ref=q["xr"])
        rec = em.rollout_feedback_tape(Z0, T, **law, xi=q["xi0"], opts=opts)
        X, U = rec["X_traj"], rec["U"]
        return 0.5 * ((X[:, :, 0] - target) ** 2).sum(axis=0) + 0.5 * 1e-2 * (U[:, :, 0] ** 2).sum(axis=0), rec, law, X, U

    L0, rec, law, X, U = loss_of(p)
    gX = np.zeros_like(X)
    gX[:, :, 0] = X[:, :, 0] - target
    g = em.rollout_feedback_vjp(rec, **law, gX=gX, gUa=1e-2 * U, slots_grad=2)
    assert (g["status"] == 0).all()
    ana = dict(kp=g["K"][0, :, 0, 0], kd=g["K"][0, :, 0, 1], ki=g["K_i"][0, :, 0, 0], xi0=g["gxi0"], xr=g["x_ref"][0])
    for k, v in p.items():
        flat = v.reshape(B, -1)
        for j in range(flat.shape[1]):
            if k == "xi0" and j == 1:
                continue  # the velocity integral has zero gain
            eps = 1e-5 * max(1.0, np.abs(flat[:, j]).max())
            qp, qm = {kk: vv.copy() for kk, vv in p.items()}, {kk: vv.copy() for kk, vv in p.items()}
            qp[k].reshape(B, -1)[:, j] += eps
            qm[k].reshape(B, -1)[:, j] -= eps
            fd = (loss_of(qp)[0] - loss_of(qm)[0]) / (2 * eps)
            an = ana[k].reshape(B, -1)[:, j]
            assert np.all(np.abs(an - fd) <= 1e-6 * np.maximum(np.abs(fd), 1e-3)), (k, j, an, fd)


def test_cartpole_gain_central_differences():
    """dL / d K_t and d u_ref_t of a cartpole with a full time-varying law against central differences"""
    m = _mech("cartpole")
    em = _emu(m)
    B, T = 1, 8
    opts = capi.solver_options(rtol=1e-11, btol=1e-11)
    Z0 = _start(m, B, 63)
    law = _law(m, T, B, 64)
    w = np.random.default_rng(65).normal(size=(T + 1, B, 2 * m.nu))

    def loss_of(lw):
        rec = em.rollout_feedback_tape(Z0, T, **lw, opts=opts)
        return float((w * rec["X_traj"]).sum() + 0.5 * (rec["U"] ** 2).sum()), rec

    _, rec = loss_of(law)
    g = em.rollout_feedback_vjp(rec, **law, gX=w, gUa=rec["U"], slots_grad=2)
    rng = np.random.default_rng(66)
    for k in ("K", "u_ref"):
        for _ in range(6):
            idx = tuple(rng.integers(0, s) for s in law[k].shape)
            eps = 1e-5
            lp, lm = {kk: vv.copy() for kk, vv in law.items()}, {kk: vv.copy() for kk, vv in law.items()}
            lp[k][idx] += eps
            lm[k][idx] -= eps
            fd = (loss_of(lp)[0] - loss_of(lm)[0]) / (2 * eps)
            an = g[k][idx]
            assert abs(an - fd) <= 1e-6 * max(abs(fd), 1e-3), (k, idx, an, fd)


def _case(name, B, T, seed, integral=True, tiled=True):
    m = _mech(name)
    em = _emu(m)
    Z0 = _start(m, B, seed)
    law = _law(m, T, B, seed + 1, integral, tiled)
    rec = em.rollout_feedback_tape(Z0, T, **law)
    gZ, gX, gUa = _cotangents(m, T, B, seed + 2)
    return em, rec, law, gZ, gX, gUa


def _same(a, b):
    return all(np.array_equal(a[k], b[k], equal_nan=True) for k in a if a[k] is not None)


@pytest.mark.parametrize("name", ("ant", "block_linear"))
def test_slots_placement_and_batch_are_bit_identical(name):
    """1 / 2 / 4 slots per CTA, both plan placements, and environment e of a batch of 8 against e run alone"""
    B, T = 8, 3
    em, rec, law, gZ, gX, gUa = _case(name, B, T, 71)
    kw = dict(gZ=gZ, gX=gX, gUa=gUa)
    ref = em.rollout_feedback_vjp(rec, **law, **kw, slots_grad=1, grid=1)
    for slots, grid in ((2, 3), (4, 1)):
        assert _same(em.rollout_feedback_vjp(rec, **law, **kw, slots_grad=slots, grid=grid), ref), (name, slots)
    assert _same(em.rollout_feedback_vjp(rec, **law, **kw, slots_grad=1, grid=1, smem_plan=False), ref), (name, "plan in global memory")
    for e in (0, 5):
        one_rec = {k: (None if v is None else (v[:, e:e + 1].copy() if v.ndim == 3 else v[e:e + 1].copy())) for k, v in rec.items()}
        one_law = {k: v[:, e:e + 1].copy() for k, v in law.items()}
        one = em.rollout_feedback_vjp(one_rec, **one_law, gZ=gZ[:, e:e + 1], gX=gX[:, e:e + 1], gUa=gUa[:, e:e + 1], slots_grad=2)
        for k in ("K", "K_i", "x_ref", "u_ref"):
            assert np.array_equal(one[k][:, 0], ref[k][:, e]), (name, e, k)
        assert np.array_equal(one["gZ0"][0], ref["gZ0"][e]) and np.array_equal(one["gxi0"][0], ref["gxi0"][e]), (name, e)


ORDERS = r"""
import sys, numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests")
from test_rollout_feedback_vjp import _case
out = {}
for name in ("ant", "block_linear"):
    em, rec, law, gZ, gX, gUa = _case(name, 4, 3, 81)
    res = em.rollout_feedback_vjp(rec, **law, gZ=gZ, gX=gX, gUa=gUa, slots_grad=2, grid=2)
    for k, v in list(res.items()) + [("tape", rec["tape"]), ("X", rec["X_traj"])]:
        out[f"{name}_{k}"] = v
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
    """HOSTEMU_ORDER=reverse|random: a race in the law stage, the per-joint scratch of M' w or its fold would show here"""
    ref = _run_order(None, str(tmp_path / "asc.npz"))
    for order in ("reverse", "random"):
        got = _run_order(order, str(tmp_path / (order + ".npz")))
        for k in ref.files:
            assert np.array_equal(ref[k], got[k], equal_nan=True), (order, k)


def test_shared_and_tiled_law_arrays():
    """steps = 1: the gradient is the sum over t, in descending order, of the tiled per-step gradients; envs = 1: per-environment
    outputs identical to a law tiled over the environments"""
    m = _mech("cartpole")
    em = _emu(m)
    B, T = 3, 5
    Z0 = _start(m, B, 91)
    shared = _law(m, T, B, 92, integral=True, tiled=False)
    tiled = {k: np.ascontiguousarray(np.broadcast_to(v, (T, B) + v.shape)) for k, v in shared.items()}
    rec = em.rollout_feedback_tape(Z0, T, **shared)
    gZ, gX, gUa = _cotangents(m, T, B, 93)
    a = em.rollout_feedback_vjp(rec, **shared, gZ=gZ, gX=gX, gUa=gUa, slots_grad=2)
    b = em.rollout_feedback_vjp(rec, **tiled, gZ=gZ, gX=gX, gUa=gUa, slots_grad=2)
    assert np.array_equal(a["gZ0"], b["gZ0"]) and np.array_equal(a["gxi0"], b["gxi0"])
    for k in ("K", "K_i", "x_ref", "u_ref"):
        s = np.zeros_like(b[k][0])
        for t in range(T - 1, -1, -1):
            s = s + b[k][t]
        assert a[k].shape[0] == 1 and np.array_equal(a[k][0], s), k
    per_env = {k: np.ascontiguousarray(np.broadcast_to(v, (B,) + v.shape)) for k, v in shared.items()}
    c = em.rollout_feedback_vjp(rec, **per_env, gZ=gZ, gX=gX, gUa=gUa, slots_grad=2)
    assert _same(a, c)


def test_nonfinite_factorisation_is_confined_to_its_environment():
    """a NaN in the tape of environment 1: status 3 and NaN in every output of that environment; the others as without it"""
    em, rec, law, gZ, gX, gUa = _case("cartpole", 3, 4, 95)
    kw = dict(gZ=gZ, gX=gX, gUa=gUa, slots_grad=2, grid=2)
    ref = em.rollout_feedback_vjp(rec, **law, **kw)
    bad = dict(rec, tape=rec["tape"].copy())
    bad["tape"][1, 1, :] = np.nan
    got = em.rollout_feedback_vjp(bad, **law, **kw)
    assert got["status"].tolist() == [0, 3, 0]
    for k in ("gZ0", "gxi0", "K", "K_i", "x_ref", "u_ref"):
        g, r = got[k], ref[k]
        axis = 0 if k in ("gZ0", "gxi0") else 1
        bad_e = np.take(g, 1, axis=axis)
        assert np.isnan(bad_e).all(), k
        for e in (0, 2):
            assert np.array_equal(np.take(g, e, axis=axis), np.take(r, e, axis=axis)), (k, e)


def test_feedback_grad_struct_matches_header():
    """the ctypes layout of DojoFeedbackGrad against include/dojo_b200.h"""
    text = open(os.path.join(ROOT, "include", "dojo_b200.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} DojoFeedbackGrad;", text).group(1)
    fields = re.findall(r"double\*\s+(\w+);", body)
    assert fields == [f for f, _ in capi.DojoFeedbackGrad._fields_] == ["K", "K_i", "x_ref", "u_ref"]
    assert ctypes.sizeof(capi.DojoFeedbackGrad) == 4 * 8


# ----------------------------------------------------------------------------------------------------- descent
# The GPU descent test's bound on final / initial loss.  The same loop (pid_descent with its defaults: 32 pendulums, T = 40, 8 iterations,
# the same seeds) ends at 0.8778 of the initial loss on the emulation, with every one of its 256 steps accepted; the bound leaves room for
# the device's rounding but not for a loop that stalls (a zero or wrong-signed gradient leaves the loss at 1.0 of where it started).
DESCENT_FRACTION = 0.9
DESCENT_T = 40


def pendulum_pid_loss(X, U):
    """per environment: the angle's squared distance to 0.5 rad over the trajectory plus a small input penalty"""
    return 0.5 * ((X[:, :, 0] - 0.5) ** 2).sum(axis=0) + 0.5e-3 * (U[:, :, 0] ** 2).sum(axis=0)


def pid_descent(rollout, vjp, B=32, iters=8, seed=101):
    """per-environment PID gains of B pendulums tuned by gradient with backtracking on pendulum_pid_loss.  rollout(law, xi0) -> rec (the
    tape's dict); vjp(rec, law, gX, gUa) -> gradients.  Each iteration re-runs the rollout at the parameters it keeps and checks, per
    environment, that an accepted step lowered the loss and a rejected one left it unchanged.  Returns (initial loss, final loss, that
    check held at every iteration, number of accepted steps)."""
    rng = np.random.default_rng(seed)
    th = np.stack([rng.uniform(1, 3, B), rng.uniform(0.0, 0.5, B), rng.uniform(0.1, 0.5, B)], axis=-1)  # kp, ki, kd
    xr = np.zeros((B, 2))
    xr[:, 0] = 0.5

    def run(th):
        law = dict(K=np.stack([th[:, 0], th[:, 2]], -1)[:, None, :], K_i=np.stack([th[:, 1], np.zeros(B)], -1)[:, None, :], x_ref=xr)
        rec = rollout(law, np.zeros((B, 2)))
        return pendulum_pid_loss(rec["X_traj"], rec["U"]), rec, law

    loss, rec, law = run(th)
    L0 = loss.sum()
    monotone, accepted = True, 0
    step = np.full(B, 1e-2)
    for _ in range(iters):
        X, U = rec["X_traj"], rec["U"]
        gX = np.zeros_like(X)
        gX[:, :, 0] = X[:, :, 0] - 0.5
        g = vjp(rec, law, gX, 1e-3 * U)
        grad = np.stack([g["K"][0, :, 0, 0], g["K_i"][0, :, 0, 0], g["K"][0, :, 0, 1]], axis=-1)
        lr = step.copy()
        for k in range(8):  # backtracking per environment: halve the step of every environment whose candidate did not lower its loss
            lc = run(th - lr[:, None] * grad)[0]
            if (lc < loss).all() or k == 7:
                break
            lr = np.where(lc < loss, lr, 0.5 * lr)
        acc = lc < loss
        accepted += int(acc.sum())
        th = np.where(acc[:, None], th - lr[:, None] * grad, th)
        new, rec, law = run(th)
        monotone &= bool(np.all(new[acc] < loss[acc]) and np.array_equal(new[~acc], loss[~acc]))
        step = np.where(acc, 1.5 * lr, 0.5 * lr)
        loss = new
    return L0, loss.sum(), monotone, accepted


def test_pid_descent_on_emulation():
    """the GPU descent loop, unchanged, on the emulation: it fixes DESCENT_FRACTION"""
    m = _mech("pendulum")
    em = _emu(m)

    def rollout(law, xi0):
        return em.rollout_feedback_tape(np.tile(m.z0, (xi0.shape[0], 1)), DESCENT_T, **law, xi=xi0)

    def vjp(rec, law, gX, gUa):
        return em.rollout_feedback_vjp(rec, **law, gX=gX, gUa=gUa, slots_grad=2)

    L0, L1, monotone, accepted = pid_descent(rollout, vjp)
    print(f"descent on the emulation: final / initial loss {L1 / L0:.4f}, {accepted} accepted steps")
    assert monotone and accepted > 0 and L1 < DESCENT_FRACTION * L0, (L0, L1, accepted)
