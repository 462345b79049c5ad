"""Reverse mode through a closed-loop rollout on the H100 (dojo_rollout_feedback_tape / dojo_rollout_feedback_vjp).

The CPU twin on the kernel emulation is tests/test_rollout_feedback_vjp.py; this file checks the device code against the dense closed-loop
recursion built from dojo_rollout_grad's Jacobians and dojo_maximal_to_minimal_jacobian on the same device, the tape against the
rollouts, the pointer kinds, the refusals and one gradient-descent problem solved with these gradients alone.
"""
import ctypes as C

import numpy as np
import pytest

from dojo_jl_b200 import capi
from dojo_jl_b200.solver import BatchedStepper
from test_rollout_feedback_vjp import DESCENT_FRACTION, DESCENT_T, _law, _mech, _start, assert_close, dense_recursion, pid_descent

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

EINVAL = -1  # DOJO_EINVAL of include/dojo_b200.h
GPU_TOL = {"ant": 1e-6, "quadruped": 1e-6, "atlas": 1e-6, "block_linear": 1e-10}


def _setup(name, B, T, seed, integral=True):
    m = _mech(name)
    s = BatchedStepper(m, B, 0)
    Z0 = _start(m, B, seed)
    law = _law(m, T, B, seed + 1, integral)
    rng = np.random.default_rng(seed + 2)
    cot = dict(gZ=rng.normal(size=(T + 1, B, 12 * m.Nb)), gX=rng.normal(size=(T + 1, B, 2 * m.nu)), gU=rng.normal(size=(T, B, m.nu)))
    return m, s, Z0, law, cot


@pytest.mark.parametrize("name", ("ant", "quadruped", "atlas", "block_linear"))
def test_matches_dense_recursion(name):
    B, T = 64, 12
    m, s, Z0, law, cot = _setup(name, B, T, 201)
    rec = s.rollout_feedback_tape(Z0, T, **law)
    got = s.rollout_feedback_vjp(rec, **law, **cot)
    assert (got["status"] == 0).all(), got["status"]
    ref, bnd = dense_recursion(m, rec, law, cot["gZ"], cot["gX"], cot["gU"], lambda Z0, U, T: s.rollout_grad(Z0, U, T)[1:3],
                               s.maximal_to_minimal_jacobian)
    for k in ("gZ0", "gxi0", "K", "K_i", "x_ref", "u_ref"):
        assert_close(got[k], ref[k], bnd[k], f"{name} {k}", GPU_TOL[name])
    s.close()


@pytest.mark.parametrize("name", ("ant", "block_linear"))
def test_tape_matches_rollouts(name):
    """Z_traj / U_applied / xi / worst status equal dojo_rollout_feedback's; Z_traj / tape / status / iterations dojo_rollout_tape's"""
    B, T = 64, 8
    m, s, Z0, law, _ = _setup(name, B, T, 211)
    rec = s.rollout_feedback_tape(Z0, T, **law)
    Zf, st_any, traj, Ua, xi = s.rollout_feedback(Z0, T, **law, record=True)
    assert np.array_equal(rec["Z_traj"][1:], traj) and np.array_equal(rec["Z_traj"][-1], Zf) and np.array_equal(rec["U"], Ua)
    assert np.array_equal(rec["xi"], xi) and np.array_equal(rec["status"].max(axis=0), st_any)
    traj2, tape2, st2, it2 = s.rollout_tape(Z0, rec["U"], T)
    assert np.array_equal(rec["Z_traj"], traj2) and np.array_equal(rec["tape"], tape2)
    assert np.array_equal(rec["status"], st2) and np.array_equal(rec["iters"], it2)
    X = np.stack([s.maximal_to_minimal(rec["Z_traj"][t]) for t in range(T + 1)])
    assert np.array_equal(rec["X_traj"], X)
    s.close()


def test_pointer_kinds_are_bit_identical():
    """host pointers, device pointers through the synchronous entries, and the _async entries on a torch stream"""
    B, T = 64, 6
    m, s, Z0, law, cot = _setup("ant", B, T, 221)
    rec = s.rollout_feedback_tape(Z0, T, **law)
    ref = s.rollout_feedback_vjp(rec, **law, **cot)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    nx, nu = 2 * m.nu, m.nu
    K = dev(np.swapaxes(law["K"], -1, -2)); Ki = dev(np.swapaxes(law["K_i"], -1, -2)); xr = dev(law["x_ref"]); ur = dev(law["u_ref"])
    dZ0 = dev(Z0)
    for kind in ("sync", "async"):
        Zt = torch.empty((T + 1, B, m.nz), dtype=torch.float64, device="cuda")
        X = torch.empty((T + 1, B, nx), dtype=torch.float64, device="cuda")
        Xi = torch.empty((T, B, nx), dtype=torch.float64, device="cuda")
        Ua = torch.empty((T, B, nu), dtype=torch.float64, device="cuda")
        tape = torch.empty((T, B, m.nres), dtype=torch.float64, device="cuda")
        st = torch.empty((T, B), dtype=torch.int32, device="cuda")
        xi = torch.zeros((B, nx), dtype=torch.float64, device="cuda")
        gZ0 = torch.empty((B, 12 * m.Nb), dtype=torch.float64, device="cuda")
        gxi0 = torch.empty((B, nx), dtype=torch.float64, device="cuda")
        gK = torch.empty((T, B, nx, nu), dtype=torch.float64, device="cuda"); gKi = torch.empty_like(gK)
        gxr = torch.empty((T, B, nx), dtype=torch.float64, device="cuda"); gur = torch.empty((T, B, nu), dtype=torch.float64, device="cuda")
        vst = torch.empty(B, dtype=torch.int32, device="cuda")
        dgZ, dgX, dgU = dev(cot["gZ"]), dev(cot["gX"]), dev(cot["gU"])
        p = lambda t: t.data_ptr()  # noqa: E731
        if kind == "async":
            stream = torch.cuda.current_stream().cuda_stream
            s.rollout_feedback_tape_device(p(dZ0), p(Zt), p(X), p(Ua), p(tape), B, T, p(K), steps=T, envs=B, dK_i=p(Ki), dx_ref=p(xr),
                                           du_ref=p(ur), dxi=p(xi), dXi_traj=p(Xi), dstatus=p(st), stream=stream)
            s.rollout_feedback_vjp_device(p(Zt), p(X), p(Ua), p(tape), p(gZ0), B, T, p(K), steps=T, envs=B, dK_i=p(Ki), dx_ref=p(xr),
                                          du_ref=p(ur), dXi_traj=p(Xi), dgZ=p(dgZ), dgX=p(dgX), dgU=p(dgU), dgK=p(gK), dgK_i=p(gKi),
                                          dgx_ref=p(gxr), dgu_ref=p(gur), dgxi0=p(gxi0), dstatus=p(vst), stream=stream)
            torch.cuda.synchronize()
        else:
            cp = lambda t: C.cast(C.c_void_p(t.data_ptr()), capi.c_double_p)  # noqa: E731
            fb = capi.DojoFeedback(T, B, cp(K), cp(Ki), cp(xr), cp(ur))
            o = capi.solver_options()
            vp = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
            assert s.L.dojo_rollout_feedback_tape(s.h, C.byref(o), B, T, vp(dZ0), C.byref(fb), vp(xi), vp(Zt), vp(X), vp(Xi), vp(Ua), vp(tape),
                                                  vp(st), None) == 0
            g = capi.DojoFeedbackGrad(cp(gK), cp(gKi), cp(gxr), cp(gur))
            assert s.L.dojo_rollout_feedback_vjp(s.h, B, T, C.byref(fb), vp(Zt), vp(X), vp(Xi), vp(Ua), vp(tape), vp(dgZ), vp(dgX), vp(dgU),
                                                 C.byref(g), vp(gZ0), vp(gxi0), vp(vst)) == 0
        assert np.array_equal(Zt.cpu().numpy(), rec["Z_traj"]) and np.array_equal(tape.cpu().numpy(), rec["tape"]), kind
        assert np.array_equal(X.cpu().numpy(), rec["X_traj"]) and np.array_equal(Xi.cpu().numpy(), rec["Xi_traj"]), kind
        assert np.array_equal(gZ0.cpu().numpy(), ref["gZ0"]) and np.array_equal(gxi0.cpu().numpy(), ref["gxi0"]), kind
        assert np.array_equal(gK.cpu().numpy().swapaxes(-1, -2), ref["K"]) and np.array_equal(gKi.cpu().numpy().swapaxes(-1, -2), ref["K_i"]), kind
        assert np.array_equal(gxr.cpu().numpy(), ref["x_ref"]) and np.array_equal(gur.cpu().numpy(), ref["u_ref"]), kind
        assert np.array_equal(vst.cpu().numpy(), ref["status"]), kind
    s.close()


def test_refusals():
    """DOJO_EINVAL before any launch: missing X_traj / tape / gZ0, Xi_traj without K_i or K_i without Xi_traj / gxi0"""
    B, T = 4, 3
    m, s, Z0, law, cot = _setup("pendulum", B, T, 231)
    rec = s.rollout_feedback_tape(Z0, T, **law)
    nx = 2 * m.nu
    L, h = s.L, s.h
    Kc = np.ascontiguousarray(np.swapaxes(law["K"], -1, -2)); Kic = np.ascontiguousarray(np.swapaxes(law["K_i"], -1, -2))
    fb = capi.DojoFeedback(T, B, capi.dptr(Kc), capi.dptr(Kic), None, None)
    fb0 = capi.DojoFeedback(T, B, capi.dptr(Kc), None, None, None)
    o = capi.solver_options()
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
    Zt, X, Xi, Ua, tape = (np.empty_like(rec[k]) for k in ("Z_traj", "X_traj", "Xi_traj", "U", "tape"))
    xi = np.zeros((B, nx))
    tapecall = lambda f, X_, Xi_, tape_: L.dojo_rollout_feedback_tape(h, C.byref(o), B, T, p(Z0), C.byref(f), p(xi), p(Zt), p(X_), p(Xi_), p(Ua),  # noqa: E731
                                                                      p(tape_), None, None)
    assert tapecall(fb, None, Xi, tape) == EINVAL
    assert tapecall(fb, X, Xi, None) == EINVAL
    assert tapecall(fb, X, None, tape) == EINVAL
    assert tapecall(fb0, X, Xi, tape) == EINVAL
    gZ0, gxi0 = np.empty((B, 12 * m.Nb)), np.empty((B, nx))
    vjpcall = lambda f, Xi_, gZ0_, gxi0_: L.dojo_rollout_feedback_vjp(h, B, T, C.byref(f), p(rec["Z_traj"]), p(rec["X_traj"]), p(Xi_),  # noqa: E731
                                                                     p(rec["U"]), p(rec["tape"]), None, None, None, None, p(gZ0_), p(gxi0_), None)
    assert vjpcall(fb, rec["Xi_traj"], None, gxi0) == EINVAL
    assert vjpcall(fb, rec["Xi_traj"], gZ0, None) == EINVAL
    assert vjpcall(fb, None, gZ0, gxi0) == EINVAL
    assert vjpcall(fb0, rec["Xi_traj"], gZ0, None) == EINVAL
    assert vjpcall(fb, rec["Xi_traj"], gZ0, gxi0) == 0
    s.close()


def test_pid_descent():
    """per-environment PID gains of 32 pendulums tuned by gradient with backtracking: every accepted step lowers the loss, and the final
    loss is below DESCENT_FRACTION of the initial one (fixed by the same loop on the emulation)"""
    m = _mech("pendulum")
    s = BatchedStepper(m, 32, 0)

    def rollout(law, xi0):
        return s.rollout_feedback_tape(np.tile(m.z0, (xi0.shape[0], 1)), DESCENT_T, **law, xi=xi0)

    def vjp(rec, law, gX, gUa):
        return s.rollout_feedback_vjp(rec, **law, gX=gX, gU=gUa)

    L0, L1, monotone, accepted = pid_descent(rollout, vjp)
    print(f"descent on the device: final / initial loss {L1 / L0:.4f}, {accepted} accepted steps")
    assert monotone and accepted > 0 and L1 < DESCENT_FRACTION * L0, (L0, L1, accepted)
    s.close()


@pytest.mark.parametrize("shared", (False, True))
def test_autograd_matches_dense_recursion(shared):
    """autograd.rollout_feedback: Z0.grad (quaternion cotangents mapped as autograd.rollout does) and every law tensor's gradient, summed
    over its broadcast dimensions, against the dense recursion"""
    from dojo_jl_b200.autograd import from_attitude, rollout_feedback, to_attitude
    name, B, T = "quadruped", 16, 8
    m, s, Z0, law, _ = _setup(name, B, T, 241)
    if shared:  # K shared by all steps and environments, x_ref per environment, u_ref per step for all environments
        law = dict(K=law["K"][0, 0], K_i=law["K_i"][0, 0], x_ref=law["x_ref"][0], u_ref=law["u_ref"][:, :1].copy())
    rng = np.random.default_rng(242)
    cZ, cX, cU = rng.normal(size=(T + 1, B, m.nz)), rng.normal(size=(T + 1, B, 2 * m.nu)), rng.normal(size=(T, B, m.nu))
    xi0 = rng.normal(0.0, 0.1, (B, 2 * m.nu))
    cu = lambda a: torch.tensor(a, dtype=torch.float64, device="cuda", requires_grad=True)  # noqa: E731
    tz, tl, txi = cu(Z0), {k: cu(v) for k, v in law.items()}, cu(xi0)
    Zt, Xt, Ut = rollout_feedback(m, tz, tl["K"], u_ref=tl["u_ref"], x_ref=tl["x_ref"], K_i=tl["K_i"], xi0=txi, T=T)
    loss = (Zt * torch.from_numpy(cZ).cuda()).sum() + (Xt * torch.from_numpy(cX).cuda()).sum() + (Ut * torch.from_numpy(cU).cuda()).sum()
    loss.backward()
    rec = s.rollout_feedback_tape(Z0, T, **law, xi=xi0)
    assert np.array_equal(Zt.detach().cpu().numpy(), rec["Z_traj"]) and np.array_equal(Ut.detach().cpu().numpy(), rec["U"])
    gZ = to_attitude(rec["Z_traj"], cZ)
    ref, bnd = dense_recursion(m, rec, law, gZ, cX, cU, lambda Z0_, U, T_: s.rollout_grad(Z0_, U, T_)[1:3], s.maximal_to_minimal_jacobian)
    tol = GPU_TOL["quadruped"]
    bZ = np.repeat(bnd["gZ0"].max(axis=-1, keepdims=True), m.nz, axis=-1)  # G(q) mixes the attitude entries: the vector's bound for all
    assert_close(tz.grad.cpu().numpy(), from_attitude(Z0, ref["gZ0"]), bZ, "Z0", tol)
    assert_close(txi.grad.cpu().numpy(), ref["gxi0"], bnd["gxi0"], "xi0", tol)
    for k, v in law.items():
        r, bd = ref[k], bnd[k]  # [T, B, *tail]
        lead = v.ndim - (2 if k in ("K", "K_i") else 1)
        if lead == 0:
            r, bd = r.sum(axis=(0, 1)), bd.sum(axis=(0, 1))
        elif lead == 1:
            r, bd = r.sum(axis=0), bd.sum(axis=0)
        elif v.shape[1] == 1:
            r, bd = r.sum(axis=1, keepdims=True), bd.sum(axis=1, keepdims=True)
        got = tl[k].grad.cpu().numpy()
        assert got.shape == v.shape, (k, got.shape, v.shape)
        assert_close(got.reshape(1, 1, -1), r.reshape(1, 1, -1), bd.reshape(1, 1, -1), f"{k} shared={shared}", tol)
    s.close()


def test_api_feedback_vjp_sums_shared_arrays():
    """api.get_feedback_vjp: gradients shaped like the law's arrays, a shared array's gradient the sum of the per-environment ones"""
    from dojo_jl_b200 import api
    name, B, T = "cartpole", 8, 10
    m, s, Z0, law, cot = _setup(name, B, T, 251)
    shared = dict(K=law["K"][0, 0], K_i=law["K_i"][0, 0], x_ref=law["x_ref"][0], u_ref=law["u_ref"][0, 0])  # x_ref per environment
    res = api.get_feedback_vjp(m, Z0, api.LinearFeedback(shared["K"], shared["x_ref"], shared["u_ref"], shared["K_i"]), T, gZ=cot["gZ"],
                               gX=cot["gX"], gU=cot["gU"])
    rec = s.rollout_feedback_tape(Z0, T, **shared)
    per = s.rollout_feedback_vjp(rec, **shared, **cot)
    assert np.array_equal(res["gZ0"], per["gZ0"])
    for k, v in shared.items():
        assert res[k].shape == np.shape(v), k
        ref = per[k][0] if np.ndim(v) == per[k].ndim - 1 else per[k][0].sum(axis=0)  # steps = 1; a shared array sums the environments
        assert np.array_equal(res[k], ref), k
    s.close()
