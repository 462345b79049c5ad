"""The inputs' configuration derivative in the step Jacobians (SURVEY.md Q17) -- CPU tests.  The GPU twin is
tests/test_zzzzzzzzz_gpu_input_jacobians.py.

An input acting between an actuated joint's two bodies is an impulse that depends on their poses.  The reference's data Jacobian
(gradients/data.jl) leaves d(input impulse)/d(x2, q2) out, so its Fz is not the derivative of its own step once a joint with a free
parent is actuated.  The library includes the term; DOJO_FLAG_Q17_LITERAL_INPUT_JACOBIAN reproduces the reference's omission.

 * first-order check of the iLQR pieces: the minimal Jacobians feed the Riccati pass, whose predicted first-order change dV1 of the
   cost must match the closed-loop rollout of the feedback law it returns: (J(a) - J(0)) / (a dV1) -> 1 linearly in a;
 * the flag: the emulated gradient kernel equals the oracle with and without it, in both compilations, and it only matters at
   nonzero inputs.
"""
import numpy as np
import pytest

import dojo_jl_b200 as dj
from dojo_jl_b200 import capi
from oracle.oracle import Oracle

from conftest import random_inputs
from test_lqr_backward import Cost, riccati
from test_oracle_properties import _lift, _random_minimal

Q17 = 4  # DOJO_FLAG_Q17_LITERAL_INPUT_JACOBIAN
Q2 = 2   # DOJO_FLAG_Q2_LITERAL_GRADIENTS
ALPHAS = (1e-2, 1e-3, 1e-4)


def active_inputs(mech):
    """inputs of the actuated joints (a floating base is not actuated)"""
    return np.concatenate([np.full(j.input_dimension, j.nimpulses > 0) for j in mech.joints])


def ilqr_problem(mech, T, seed):
    """airborne minimal start (every contact 3 m away), random nominal inputs on the actuated joints, a quadratic cost about goals
    away from the nominal trajectory"""
    rng = np.random.default_rng(seed)
    x0 = _random_minimal(mech, rng, 0.2, 0.5)
    x0[2] += 3.0
    U = np.stack([random_inputs(mech, 1, rng, 0.5) for _ in range(T)])  # [T, 1, nu]
    nx, nu = 2 * mech.nu, mech.nu
    cost = Cost(np.eye(nx), 0.1 * np.eye(nu), x0 + rng.normal(0.0, 0.3, (T, nx)), rng.normal(0.0, 0.5, nu),
                2.0 * np.eye(nx), x0 + rng.normal(0.0, 0.3, nx))
    return x0, U, cost


def cost_value(cost, X, U):
    """J = sum_t 1/2 |x_t - xg_t|_Q^2 + 1/2 |u_t - ug|_R^2 + 1/2 |x_T - xg_T|_Qf^2 (the cost the Riccati recursion expands)"""
    T = U.shape[0]
    J = 0.0
    for t in range(T):
        dx, du = X[t] - cost.x_goal[t], U[t] - cost.u_goal
        J += 0.5 * dx @ cost.Q @ dx + 0.5 * du @ cost.R @ du
    dx = X[T] - cost.x_goal_final
    return J + 0.5 * dx @ cost.Q_final @ dx


def first_order_ratios(Gx, Gu, X, U, cost, rollout, active):
    """lqr_backward on the Jacobians, then J(a) of the closed loop u = U + a k - K (x - X); returns (J(a) - J(0)) / (a dV1) per a"""
    T = U.shape[0]
    K, k, dV, status = riccati(X[:, None], U[:, None], Gx[:, None], Gu[:, None],
                               Cost(cost.Q, cost.R, cost.x_goal[:, None], cost.u_goal, cost.Q_final[None], cost.x_goal_final[None]),
                               active=active)
    assert status[0] == 0 and dV[0, 0] < 0.0
    J0 = cost_value(cost, *rollout(K[:, 0], X, U, 0.0 * k[:, 0]))
    assert abs(J0 - cost_value(cost, X, U)) <= 1e-12 * abs(J0)
    return np.array([(cost_value(cost, *rollout(K[:, 0], X, U, a * k[:, 0])) - J0) / (a * dV[0, 0]) for a in ALPHAS])


def check_first_order(r):
    """the ratio tends to 1 and its error shrinks about linearly with a (second-order term a^2 dV2 plus the curvature of the step)"""
    err = np.abs(r - 1.0)
    assert err[-1] < 2e-4, r
    assert err[1] < 0.3 * err[0] + 1e-5 and err[2] < 0.3 * err[1] + 1e-5, r


def test_ilqr_first_order_check_on_the_oracle():
    """raiberthopper: its prismatic leg's input force has a lever arm that moves along the joint (Q16's half torque), so the term
    shows in minimal coordinates too.  (A revolute joint's input torque lies on its axis, which the joint's own rotation leaves in
    place: for mechanisms of revolute joints such as ant and quadruped the term vanishes along the constraint manifold.)"""
    mech = dj.get_mechanism("raiberthopper")
    opts = capi.solver_options(rtol=1e-11, btol=1e-11)
    o = Oracle(mech, opts)
    T = 6
    x0, U, cost = ilqr_problem(mech, T, seed=21)
    U = U[:, 0]

    def rollout(K, Xref, Uref, dk):
        """host feedback loop around the oracle step, in minimal coordinates"""
        z = o.minimal_to_maximal(x0)
        X, Ua = [o.maximal_to_minimal(z)], []
        for t in range(T):
            u = Uref[t] + dk[t] - K[t] @ (X[t] - Xref[t])
            z, st, _ = o.step(z, u)
            assert st == 0
            X.append(o.maximal_to_minimal(z))
            Ua.append(u)
        return np.array(X), np.array(Ua)

    X, _ = rollout(np.zeros((T, mech.nu, 2 * mech.nu)), np.zeros((T + 1, 2 * mech.nu)), U, np.zeros_like(U))
    Gx, Gu = [], []
    for t in range(T):
        xn, gx, gu, st, _ = o.minimal_gradients(X[t], U[t])
        assert st == 0 and np.abs(xn - X[t + 1]).max() < 1e-10
        Gx.append(gx)
        Gu.append(gu)
    check_first_order(first_order_ratios(np.array(Gx), np.array(Gu), X, U, cost, rollout, active_inputs(mech)))


def _flag_case(name, seed, B=2, lift=3.0):
    if name == "block_linear":
        mech = dj.get_mechanism("block", contact_type="linear")
    else:
        mech = dj.get_mechanism(name)
    rng = np.random.default_rng(seed)
    Z = np.tile(_lift(mech.z0, lift), (B, 1))
    Z[:, 3:6] += rng.normal(0.0, 0.3, (B, 3))
    Z[:, 10:13] += rng.normal(0.0, 0.3, (B, 3))
    U = rng.uniform(-1.0, 1.0, (B, mech.nu))  # a floating base's input acts against the world frame: its torque moves with the body
    return mech, Z, U


@pytest.mark.parametrize("name,lift", [("ant", 3.0), ("ant", 0.0), ("raiberthopper", 3.0), ("raiberthopper", 0.0), ("block_linear", 0.0)])
def test_flag_emulated_kernel_matches_oracle(name, lift):
    """ant: NonlinearContact (dj); raiberthopper and the LinearContact block: the DJ_ANY_CONTACT compilation (dj_cm).  Without the
    flag the kernel carries the inputs' configuration derivative like the oracle; with it (alone or with Q2) both omit it."""
    from hostemu.harness import HostEmu
    mech, Z, U = _flag_case(name, seed=5, lift=lift)
    o, em = Oracle(mech), HostEmu(mech)
    moved = 0.0
    for flags in (0, Q17, Q2 | Q17, Q2):
        Zn, Fz, Fu, st, it = em.step_grad(Z, U, slots=2, slots_grad=2, flags=flags)
        for e in range(len(Z)):
            zo, Fzo, Fuo, so, io = o.step_grad(Z[e], U[e], flags=flags)
            assert (st[e], it[e]) == (so, io)
            assert np.abs(Zn[e] - zo).max() < 1e-10
            assert np.abs(Fz[e] - Fzo).max() < 1e-8 * max(1.0, np.abs(Fzo).max()), (flags, np.abs(Fz[e] - Fzo).max())
            assert np.abs(Fu[e] - Fuo).max() < 1e-8 * max(1.0, np.abs(Fuo).max())
        if flags == 0:
            Fz0, Fu0 = Fz, Fu
        if flags == Q17:
            # the flag changes Fz only (the input columns do not depend on it), and by the input term
            assert np.array_equal(Fu, Fu0)
            moved = np.abs(Fz - Fz0).max() / max(1.0, np.abs(Fz0).max())
    assert moved > 1e-4, moved


@pytest.mark.parametrize("name", ["ant", "raiberthopper"])
def test_flag_changes_nothing_at_zero_inputs(name):
    """at u = 0 the inputs' configuration derivative vanishes: with and without the flag the kernel returns the same numbers"""
    from hostemu.harness import HostEmu
    mech, Z, _ = _flag_case(name, seed=6)
    em = HostEmu(mech)
    U = np.zeros((len(Z), mech.nu))
    a = em.step_grad(Z, U, slots=2, slots_grad=2)
    b = em.step_grad(Z, U, slots=2, slots_grad=2, flags=Q17)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
