"""Reverse mode in minimal coordinates -- CPU suite: the adjoints of the coordinate maps (dojo_kinjac.cuh: max_to_min_vjp_env,
min_to_max_vjp_env, run with one "thread" through tests/hostcheck) and their composition with the rollout tape and adjoint on the kernel
emulation (tests/hostemu).

The reference for the rollout is the dense MAXIMAL recursion: z_0 = n(X0), z_{t+1} = step(z_t, u_t), x_t = m(z_t), built from the
emulated rollout_grad Jacobians Fz / Fu, the dense M(z_t) at every slab and N(z_0).  The chain of get_minimal_gradients (M Fz N) is the
derivative of another computation, which re-enters maximal coordinates through n(m(z_t)) at every step, and is not used here.  The -m gpu
twin is tests/test_zzzzzzzzzzzzz_gpu_minimal_vjp.py.
"""
import numpy as np
import pytest

import dojo_jl_b200 as dj
from conftest import jittered_states
from dojo_jl_b200 import capi
from test_rollout_vjp import TOL, _emu, _mech, _slots_grad, _start, assert_close, contract


def _hc(m):
    from hostcheck.minimal_vjp import MapVjp
    return MapVjp(m)


def _rel_close(got, ref, bound, what, tol):
    """|got - ref| <= tol * max over the state's vector of the absolute contraction"""
    scale = np.maximum(bound.max(axis=-1, keepdims=True), 1e-300)
    err = np.abs(got - ref) / scale
    assert np.isfinite(got).all() and err.max() <= tol, f"{what}: worst {err.max():.2e} of the bound at {np.argwhere(err > tol)[:4].tolist()}"


def _states(m, hc, rng, B=3):
    """(label, Z) test states: jittered configurations at rest; the same with random joint velocities; exactly-zero joint coordinates, at
    rest and moving; a root joint rotated by 2.5 rad, moving.  The last four are minimal_to_maximal of a minimal state."""
    nm = 2 * m.nu
    if m.Nb > 1:
        Zj = jittered_states(m, B, rng)
    else:
        Zj = np.tile(m.z0, (B, 1))
        Zj[:, 6:10] = [np.cos(0.2), np.sin(0.2) * 0.6, np.sin(0.2) * 0.8, 0.0]
    vel = np.zeros((B, nm))
    for j in m.joints:
        n = j.input_dimension
        vel[:, 2 * j_off(m, j) + n:2 * j_off(m, j) + 2 * n] = rng.normal(0.0, 1.0, (B, n))
    Xj = hc.maximal_to_minimal(Zj)
    X0 = np.zeros((B, nm))
    Xr = Xj + vel
    for j in m.joints:
        if j.parent >= 0 or j.rot.nfree == 0:
            continue
        o = 2 * j_off(m, j) + j.tra.nfree
        v = rng.normal(size=(B, j.rot.nfree))
        Xr[:, o:o + j.rot.nfree] = 2.5 * v / np.linalg.norm(v, axis=1, keepdims=True)
    return [("jittered", Zj), ("moving", hc.minimal_to_maximal(Xj + vel)), ("zero", hc.minimal_to_maximal(X0)),
            ("zero_moving", hc.minimal_to_maximal(X0 + vel)), ("root_2.5rad", hc.minimal_to_maximal(Xr))]


def j_off(m, j):
    """the joint's offset in the input vector (joint order)"""
    off = 0
    for k in m.joints:
        if k is j:
            return off
        off += k.input_dimension
    raise KeyError(j.name)


def _mechanisms():
    from hostcheck.kinjac_vjp import mechanisms
    return mechanisms()


# ----------------------------------------------------------------------------------------------------- the two map adjoints
def test_map_adjoints_match_dense_jacobians():
    """M(z)' gX and N(z)' gZ against the contraction of the dense map Jacobians of hostcheck.cpp, every mechanism and all 16 joint
    prototypes, at rest, moving, at exactly-zero joint coordinates and with a root rotated by 2.5 rad"""
    rng = np.random.default_rng(41)
    names = []
    for name, m in _mechanisms():
        names.append(name)
        hc = _hc(m)
        for label, Z in _states(m, hc, rng):
            B = Z.shape[0]
            gX, gZ = rng.normal(size=(B, 2 * m.nu)), rng.normal(size=(B, 12 * m.Nb))
            M = hc.maximal_to_minimal_jacobian(Z)
            _rel_close(hc.max_to_min_vjp(Z, gX), np.einsum("bij,bi->bj", M, gX), np.einsum("bij,bi->bj", np.abs(M), np.abs(gX)),
                       f"{name} {label} M'", 1e-13)
            N = hc.minimal_to_maximal_jacobian(Z)
            _rel_close(hc.min_to_max_vjp(Z, gZ), np.einsum("bij,bi->bj", N, gZ), np.einsum("bij,bi->bj", np.abs(N), np.abs(gZ)),
                       f"{name} {label} N'", 1e-13)
    assert "atlas" in names and sum(n.startswith("snake_") for n in names) == 16, names


def test_atlas_chain_runs_against_joint_order():
    """atlas lists children before parents (its root -> leaves order is not the joint order), so N' must walk the reverse of that order:
    a single cotangent on a leaf body reaches every joint on the path to the root"""
    m = dj.get_mechanism("atlas")
    order = list(m.root_to_leaves_joints())
    assert order != sorted(order)
    hc = _hc(m)
    Z = hc.minimal_to_maximal(np.zeros((1, 2 * m.nu)))
    leaf = m.joints[order[-1]].child
    gZ = np.zeros((1, 12 * m.Nb))
    gZ[0, 12 * leaf:12 * leaf + 12] = 1.0
    got = hc.min_to_max_vjp(Z, gZ)
    ref = np.einsum("bij,bi->bj", hc.minimal_to_maximal_jacobian(Z), gZ)
    assert np.abs(got - ref).max() <= 1e-13 * np.abs(ref).max()
    assert (np.abs(got[0, :12]) > 0).any()  # the floating base, at the root


def test_state_alone_equals_state_in_a_batch():
    """the result of state e does not depend on the other states: alone and among 7 others, bit for bit"""
    rng = np.random.default_rng(43)
    for name in ("ant", "atlas", "pendulum"):
        m = dj.get_mechanism(name)
        hc = _hc(m)
        Z = _states(m, hc, rng, B=8)[1][1]
        gX, gZ = rng.normal(size=(8, 2 * m.nu)), rng.normal(size=(8, 12 * m.Nb))
        allM, allN = hc.max_to_min_vjp(Z, gX), hc.min_to_max_vjp(Z, gZ)
        for e in (0, 5):
            assert np.array_equal(hc.max_to_min_vjp(Z[e:e + 1], gX[e:e + 1])[0], allM[e])
            assert np.array_equal(hc.min_to_max_vjp(Z[e:e + 1], gZ[e:e + 1])[0], allN[e])


# ----------------------------------------------------------------------------------------------------- composition with the rollout adjoint
def minimal_vjp(em, hc, X0, U, gX, opts=None, slots_grad=1):
    """the minimal-coordinate rollout adjoint as the library composes it: z0 = n(X0), tape, gZ[t] = M(z_t)' gX[t], rollout_vjp,
    gX0 = N(z0)' lambda_0.  Returns (traj, X_traj, gX0, gU, status, vjp status)."""
    T, B = U.shape[0], U.shape[1]
    traj, tape, st, _ = em.rollout_tape(hc.minimal_to_maximal(X0), U, T, opts, slots=2, grid=2)
    Xt = hc.maximal_to_minimal(traj.reshape(-1, traj.shape[-1])).reshape(T + 1, B, -1)
    gZ = hc.max_to_min_vjp(traj.reshape(-1, traj.shape[-1]), gX.reshape(-1, gX.shape[-1])).reshape(T + 1, B, -1)
    gZ0, gU, vst = em.rollout_vjp(traj, U, tape, gZ, slots_grad=slots_grad, grid=2)
    return traj, Xt, hc.min_to_max_vjp(traj[0], gZ0), gU, st, vst


def dense_reference(em, hc, X0, U, gX, opts=None, slots_grad=1):
    """the dense maximal recursion and its bound: gZ[t] = M_t' gX[t], the contraction of rollout_grad's Fz / Fu, gX0 = N_0' lambda_0"""
    T, B = U.shape[0], U.shape[1]
    traj, Fz, Fu, st, _ = em.rollout_grad(hc.minimal_to_maximal(X0), U, T, opts, slots=2, slots_grad=slots_grad, grid=2)
    M = hc.maximal_to_minimal_jacobian(traj.reshape(-1, traj.shape[-1])).reshape(T + 1, B, 2 * U.shape[2], -1)
    gZ = np.einsum("tbij,tbi->tbj", M, gX)
    gZa = np.einsum("tbij,tbi->tbj", np.abs(M), np.abs(gX))
    lam, gUr, _, _ = contract(Fz, Fu, gZ)
    _, _, lamA, gUa = contract(np.abs(Fz), np.abs(Fu), gZa)
    N0 = hc.minimal_to_maximal_jacobian(traj[0])
    return traj, np.einsum("bij,bi->bj", N0, lam), gUr, np.einsum("bij,bi->bj", np.abs(N0), lamA), gUa, st


@pytest.mark.parametrize("name", ("pendulum", "cartpole", "quadruped", "raiberthopper", "block_linear", "ant"))
def test_rollout_composition_matches_dense_recursion(name):
    """gX0 / gU of the composition against the dense maximal recursion, random cotangents on every slab (1e-10 of the bound; ant 1e-6,
    the floor of test_rollout_vjp).  Ant and quadruped run with a solver budget that ends some steps :failed."""
    m = _mech(name)
    em, hc = _emu(m), _hc(m)
    B, T = 3, 8 if m.Nb > 2 else 12
    Z0, U = _start(m, B, T, seed=45)
    X0 = hc.maximal_to_minimal(Z0)
    opts = capi.solver_options(max_iter=8) if name in ("ant", "quadruped") else None
    gX = np.random.default_rng(46).normal(size=(T + 1, B, 2 * m.nu))
    traj, Xt, gX0, gU, st, vst = minimal_vjp(em, hc, X0, U, gX, opts, _slots_grad(m))
    traj2, gX0r, gUr, gX0a, gUa, st2 = dense_reference(em, hc, X0, U, gX, opts, _slots_grad(m))
    assert np.array_equal(traj, traj2) and np.array_equal(st, st2) and (vst == 0).all()
    if opts is not None:
        assert (st == 1).any(), f"no step ended :failed: {st}"
    tol = TOL.get(name, 1e-10)
    assert_close(gX0, gX0r, gX0a, f"{name} gX0", tol)
    assert_close(gU, gUr, gUa, f"{name} gU", tol)


def _loss(em, hc, X0, U, d, opts):
    T = U.shape[0]
    traj, _, st, _ = em.rollout_tape(hc.minimal_to_maximal(X0), U, T, opts)
    assert (st == 0).all()
    Xt = hc.maximal_to_minimal(traj.reshape(-1, traj.shape[-1])).reshape(T + 1, 1, -1)
    return float(np.sum(d * Xt))


@pytest.mark.parametrize("name", ("pendulum", "cartpole"))
def test_central_differences(name):
    """the scalar loss sum_t d_t' x_t on the minimal trajectory, solved at rtol = btol = 1e-11: gX0 and gU against central differences"""
    m = _mech(name)
    em, hc = _emu(m), _hc(m)
    T = 6
    Z0, U = _start(m, 1, T, seed=47)
    X0 = hc.maximal_to_minimal(Z0)
    opts = capi.solver_options(rtol=1e-11, btol=1e-11, max_iter=100)
    d = np.random.default_rng(48).normal(size=(T + 1, 1, 2 * m.nu))
    _, _, gX0, gU, st, vst = minimal_vjp(em, hc, X0, U, d, opts)
    assert (st == 0).all() and vst[0] == 0
    eps = 1e-6
    fd_u = np.zeros_like(gU)
    for t in range(T):
        for j in range(m.nu):
            Up, Um = U.copy(), U.copy()
            Up[t, 0, j] += eps
            Um[t, 0, j] -= eps
            fd_u[t, 0, j] = (_loss(em, hc, X0, Up, d, opts) - _loss(em, hc, X0, Um, d, opts)) / (2 * eps)
    fd_x = np.zeros(2 * m.nu)
    for k in range(2 * m.nu):
        Xp, Xm = X0.copy(), X0.copy()
        Xp[0, k] += eps
        Xm[0, k] -= eps
        fd_x[k] = (_loss(em, hc, Xp, U, d, opts) - _loss(em, hc, Xm, U, d, opts)) / (2 * eps)
    scale = max(1.0, np.abs(fd_x).max(), np.abs(fd_u).max())
    assert np.abs(gU - fd_u).max() < 1e-6 * scale, (np.abs(gU - fd_u).max(), scale)
    assert np.abs(gX0[0] - fd_x).max() < 1e-6 * scale, (np.abs(gX0[0] - fd_x).max(), scale)


def test_ctypes_prototypes_match_header():
    """the four new entries are declared in include/dojo_b200.h with the argument lists the binding gives them"""
    import os
    import re
    from dojo_jl_b200 import solver
    text = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dojo_b200.h")).read()
    for name, nargs in (("dojo_maximal_to_minimal_vjp", 5), ("dojo_minimal_to_maximal_vjp", 5), ("dojo_maximal_to_minimal_vjp_async", 6),
                        ("dojo_minimal_to_maximal_vjp_async", 6)):
        m = re.search(r"\bint " + name + r"\(([^)]*)\);", text)
        assert m and len(m.group(1).split(",")) == nargs, name
        assert name in solver.EXPORTS
