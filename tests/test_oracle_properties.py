"""Property tests that pin the CPU oracle (oracle/) -- the reference's own test strategy restated (SURVEY.md §4):
no golden vectors exist in the reference, its tests are analytic-vs-finite-difference and conservation checks.

  test/jacobian.jl:1-117   full_matrix(system) == -d(rhs)/d(solution)       -> test_solution_matrix_matches_finite_difference
  test/data.jl:82-125      jacobian_data! == d(rhs)/d(data) * attjac          -> test_data_jacobian_matches_finite_difference
  test/momentum.jl:154-219 momentum conservation (atlas, quadruped, g = 0)    -> test_momentum_conservation
  test/joint_limits.jl     pendulum rests on its limit                         -> test_pendulum_joint_limit
  test/behaviors.jl:1-19   quadruped never penetrates                          -> test_quadruped_no_penetration
  (ours)                   block LDU == dense partial-pivot LU                 -> test_block_ldu_matches_dense_lu
  (ours)                   IFT gradients == finite differences of the step     -> test_ift_gradients_match_finite_difference
"""
import numpy as np
import pytest

import dojo_jl_b200 as dj
from dojo_jl_b200 import capi, quat as Q
from oracle.oracle import Oracle

from conftest import random_inputs

MECHS = ["pendulum", "ant", "quadruped", "atlas"]


def _advance(o, mech, z, u, steps):
    for _ in range(steps):
        z, _, _ = o.step(z, u)
    return z


@pytest.mark.parametrize("name,steps", [("pendulum", 10), ("ant", 2), ("ant", 30), ("quadruped", 2), ("quadruped", 45), ("atlas", 2), ("atlas", 40)])
def test_solution_matrix_matches_finite_difference(name, steps):
    mech = dj.get_mechanism(name)
    o = Oracle(mech, capi.solver_options(rtol=1e-7, btol=1e-7))
    u = 0.1 * np.ones(mech.nu)
    z = _advance(o, mech, mech.z0.copy(), u, steps)
    _, _, _, sol = o.step(z, u, return_sol=True)
    mu = o.trace()[-1, 3]
    mu = 0.0 if mu != mu else mu
    o.set_state(z, u)
    o.set_solution(sol, mu)
    A, _ = o.assemble(mu)
    fd = np.zeros_like(A)
    d = 1e-5
    for i in range(mech.nres):
        sp, sm = sol.copy(), sol.copy()
        sp[i] += d
        sm[i] -= d
        fd[:, i] = (o.evaluate_rhs(sp, mu) - o.evaluate_rhs(sm, mu)) / (2 * d)
    assert np.abs(fd + A).max() < 1e-6


def _perturb_state(z, i, eps):
    b, k = divmod(i, 12)
    z2 = z.copy()
    base = 13 * b
    if k < 6:
        z2[base + k] += eps
    elif k < 9:  # attitude: q + LV'(q) dphi
        q = z[base + 6:base + 10]
        dphi = np.zeros(3)
        dphi[k - 6] = eps
        z2[base + 6:base + 10] = q + Q.qmul(q, np.concatenate([[0.0], dphi]))
    else:
        z2[base + 10 + (k - 9)] += eps
    return z2


DATA_CASES = [("pendulum", 5, 1.0, 0.2), ("ant", 30, None, None), ("quadruped", 40, 0.3, 0.1), ("atlas", 3, None, None), ("cartpole", 5, None, None),
              ("raiberthopper", 5, None, None)]


@pytest.mark.parametrize("name,steps,spring,damper,u_value", [pytest.param(*c, 0.0, id="-".join(map(str, c))) for c in DATA_CASES] +
                         [pytest.param(*c, 0.5, id="-".join(map(str, c)) + "-u0.5") for c in DATA_CASES])
def test_data_jacobian_matches_finite_difference(name, steps, spring, damper, u_value):
    """test/data.jl evaluates the finite differences with zero inputs (joint.input is cleared by input_impulse!).  With
    u = 0.5 on every input the state columns also carry d(input impulse)/d(x2, q2), which the reference omits (SURVEY Q17)."""
    mech = dj.get_mechanism(name)
    if spring is not None:
        for j in mech.joints:
            if j.nimpulses:
                j.tra.spring = j.rot.spring = spring
                j.tra.damper = j.rot.damper = damper
    o = Oracle(mech, capi.solver_options(rtol=1e-8, btol=1e-8))
    u0 = 0.2 * np.ones(mech.nu)
    if mech.joints[0].nimpulses == 0:
        u0[:6] = 0
    z = _advance(o, mech, mech.z0.copy(), u0, steps)
    u = u_value * np.ones(mech.nu)
    _, _, _, sol = o.step(z, u, return_sol=True)
    mu = o.trace()[-1, 3]
    mu = 0.0 if mu != mu else mu
    o.set_state(z, u)
    o.set_solution(sol, mu)
    o.assemble(mu)
    D = o.data_jacobian()
    ns, eps = 12 * mech.Nb, 1e-6
    rng = np.random.default_rng(0)
    cols = list(range(ns + mech.nu)) if ns + mech.nu <= 200 else list(rng.choice(ns + mech.nu, 120, replace=False))
    worst = 0.0
    for i in cols:
        if i < ns:
            o.set_state(_perturb_state(z, i, eps), u)
            rp = o.evaluate_rhs(sol, mu)
            o.set_state(_perturb_state(z, i, -eps), u)
            rm = o.evaluate_rhs(sol, mu)
        else:
            up, um = u.copy(), u.copy()
            up[i - ns] += eps
            um[i - ns] -= eps
            o.set_state(z, up)
            rp = o.evaluate_rhs(sol, mu)
            o.set_state(z, um)
            rm = o.evaluate_rhs(sol, mu)
        worst = max(worst, np.abs((rp - rm) / (2 * eps) - D[:, i]).max())
    assert worst < 1e-6


@pytest.mark.parametrize("name,steps", [("ant", 25), ("quadruped", 40), ("atlas", 30)])
def test_block_ldu_matches_dense_lu(name, steps):
    mech = dj.get_mechanism(name)
    o = Oracle(mech)
    u = 0.1 * np.ones(mech.nu)
    z = _advance(o, mech, mech.z0.copy(), u, steps)
    _, _, _, sol = o.step(z, u, return_sol=True)
    o.set_state(z, u)
    o.set_solution(sol, 1e-6)
    A, b = o.assemble(1e-6)
    x_ldu = o.linear_solve(b, 0)
    x_lu = o.linear_solve(b, 1)
    x_np = np.linalg.solve(A, b)
    scale = np.abs(x_np).max()
    assert np.abs(x_lu - x_np).max() / scale < 1e-9
    assert np.abs(x_ldu - x_np).max() / scale < 1e-5  # no pivoting across blocks: looser, as the reference's LDU
    assert np.abs(A @ x_ldu - b).max() < 1e-7


@pytest.mark.parametrize("name,spring,damper,steps", [("quadruped", 0.3, 0.1, 300), ("atlas", 10.0, 1.0, 200), ("ant", 1.0, 1.0, 200)])
def test_momentum_conservation(name, spring, damper, steps):
    """test/momentum.jl: g = 0, no contacts, springs + dampers + control (u = 0.5 on every non-floating joint for the first
    100 steps), rtol = btol = 1e-12, |dp| < 1e-8."""
    mech = dj.get_mechanism(name, gravity=0.0)
    mech.contacts = []
    for j in mech.joints:
        if j.nimpulses:
            j.tra.spring = j.rot.spring = spring
            j.tra.damper = j.rot.damper = damper
    o = Oracle(mech, capi.solver_options(rtol=1e-12, btol=1e-12))
    z = mech.z0.copy()
    P = []
    for k in range(steps):
        u = np.concatenate([(0.5 if (j.input_dimension <= 5 and k < 100) else 0.0) * np.ones(j.input_dimension) for j in mech.joints])
        z, st, _ = o.step(z, u)
        assert st == 0
        P.append(o.momentum())
    P = np.array(P)
    assert np.abs(P - P[0]).max() < 1e-8


def test_pendulum_joint_limit():
    """test/joint_limits.jl: the pendulum comes to rest on its joint limit."""
    mech = dj.get_mechanism("pendulum")
    j = mech.joints[0]
    j.rot.limit_lo, j.rot.limit_hi = np.array([0.25 * np.pi]), np.array([np.pi])
    j.tra.damper = j.rot.damper = 0.5  # bleed the energy so that it settles quickly
    mech.z0 = mech.forward_kinematics({"joint": [0.4 * np.pi]})
    o = Oracle(mech)
    z = mech.z0.copy()
    for _ in range(1500):
        z, st, _ = o.step(z, np.zeros(1))
    th = mech.minimal_coordinates(z)["joint"][0]
    assert abs(th - 0.25 * np.pi) < 1e-3


def test_quadruped_no_penetration():
    """test/behaviors.jl:1-19: contact sdf >= 0 (to solver tolerance) while the quadruped falls and settles."""
    mech = dj.get_mechanism("quadruped")
    o = Oracle(mech)
    z = mech.z0.copy()
    worst = 1.0
    for _ in range(120):
        z, st, _ = o.step(z, np.zeros(mech.nu))
        x, _, q, _ = dj.unpack_maximal_state(z)
        for c in mech.contacts:
            sdf = c.normal @ (x[c.body] + Q.qrot(c.origin, q[c.body]) - c.offset) - c.radius
            worst = min(worst, sdf)
    assert worst > -1e-3


def _reduce(zz, zref, Nb):
    out = []
    for b in range(Nb):
        a, r = zz[13 * b:13 * b + 13], zref[13 * b:13 * b + 13]
        dq = Q.qmul(Q.qconj(r[6:10]), a[6:10])
        out += [a[0:3] - r[0:3], a[3:6] - r[3:6], dq[1:4], a[10:13] - r[10:13]]
    return np.concatenate(out)


def _lift(z, height):
    z = z.copy().reshape(-1, 13)
    z[:, 2] += height
    return z.reshape(-1)


# (mechanism, roll-in steps from z0 with u = 0, lift of every body before the roll-in, input scale, solver tolerance)
IFT_CASES = [pytest.param("pendulum", 10, 0.0, 0.0, 1e-10, id="pendulum-10"), pytest.param("ant", 3, 0.0, 0.0, 1e-10, id="ant-3"),
             pytest.param("pendulum", 10, 0.0, 1.0, 1e-10, id="pendulum-10-u1"), pytest.param("ant", 3, 0.0, 1.0, 1e-10, id="ant-3-u1"),
             pytest.param("ant", 2, 3.0, 1.0, 1e-10, id="ant-airborne-u1"), pytest.param("quadruped", 2, 3.0, 1.0, 1e-10, id="quadruped-airborne-u1"),
             pytest.param("raiberthopper", 2, 3.0, 1.0, 1e-10, id="raiberthopper-airborne-u1"),
             pytest.param("quadruped", 40, 0.0, 0.3, 1e-11, id="quadruped-sticking-u0.3")]  # settled on sticking contacts


@pytest.mark.parametrize("name,steps,lift,u_scale,tol", IFT_CASES)
def test_ift_gradients_match_finite_difference(name, steps, lift, u_scale, tol):
    """get_maximal_gradients (consistent IFT at the solution, SURVEY Q2) vs central differences of the step itself, at zero and at
    random nonzero inputs U(-u_scale, u_scale) on the actuated joints: Fz includes d(input impulse)/d(x2, q2) (SURVEY Q17), which
    the reference's data Jacobian omits.  The airborne cases lift the whole mechanism 3 m, so no contact is active."""
    mech = dj.get_mechanism(name)
    o = Oracle(mech, capi.solver_options(rtol=tol, btol=tol))
    u = random_inputs(mech, 1, np.random.default_rng(3), u_scale)[0]
    z = _advance(Oracle(mech), mech, _lift(mech.z0, lift), np.zeros(mech.nu), steps)
    zn, Fz, Fu, st, it0 = o.step_grad(z, u)
    _, Fz2, Fu2, _, _ = o.step_grad(z, u, use_factor=True)
    assert st == 0
    assert np.abs(Fz - Fz2).max() < 1e-4 * max(1.0, np.abs(Fz).max())
    ns, eps = 12 * mech.Nb, 1e-6
    rng = np.random.default_rng(0)
    cols = range(ns) if ns <= 24 else rng.choice(ns, 16, replace=False)
    checked = 0
    for i in cols:
        zp, _, ip = o.step(_perturb_state(z, i, eps), u)
        zm, _, im = o.step(_perturb_state(z, i, -eps), u)
        if ip != it0 or im != it0:
            continue  # a different Newton-iteration count changes the (tolerance-level) solver error: FD noise / eps
        col = (_reduce(zp, zn, mech.Nb) - _reduce(zm, zn, mech.Nb)) / (2 * eps)
        assert np.abs(col - Fz[:, i]).max() < 2e-5 * max(1.0, np.abs(Fz).max())
        checked += 1
    for i in range(mech.nu):
        up, um = u.copy(), u.copy()
        up[i] += eps
        um[i] -= eps
        zp, _, ip = o.step(z, up)
        zm, _, im = o.step(z, um)
        if ip != it0 or im != it0:
            continue
        col = (_reduce(zp, zn, mech.Nb) - _reduce(zm, zn, mech.Nb)) / (2 * eps)
        assert np.abs(col - Fu[:, i]).max() < 1e-5 * max(1.0, np.abs(Fu).max())
        checked += 1
    assert checked >= 8


# ----------------------------------------------------------------------------------------------------------------
# minimal <-> maximal coordinate maps (SURVEY.md 8 f1; reference test/minimal.jl: the maps are mutual inverses)
# ----------------------------------------------------------------------------------------------------------------
def _random_minimal(mech, rng, scale_c=0.3, scale_v=0.5):
    x = np.zeros(2 * mech.nu)
    off = 0
    for j in mech.joints:
        n = j.input_dimension
        x[2 * off:2 * off + n] = rng.uniform(-scale_c, scale_c, n)
        x[2 * off + n:2 * off + 2 * n] = rng.normal(0.0, scale_v, n)
        off += n
    return x


@pytest.mark.parametrize("name", ["pendulum", "ant", "quadruped", "atlas"])
def test_minimal_maximal_round_trip(name):
    """maximal_to_minimal(minimal_to_maximal(x)) == x (test/minimal.jl) -- coordinates and finite-difference velocities --
    and the configuration agrees with the independently written host forward kinematics (set_minimal_coordinates!)."""
    mech = dj.get_mechanism(name)
    o = Oracle(mech)
    rng = np.random.default_rng(5)
    for _ in range(5):
        x = _random_minimal(mech, rng)
        z = o.minimal_to_maximal(x)
        assert np.abs(o.maximal_to_minimal(z) - x).max() < 1e-10
        coords, off = {}, 0
        for j in mech.joints:
            coords[j.name] = x[2 * off:2 * off + j.input_dimension]
            off += j.input_dimension
        zk = mech.forward_kinematics(coords).reshape(mech.Nb, 13)
        zz = z.reshape(mech.Nb, 13)
        assert np.abs(zz[:, 0:3] - zk[:, 0:3]).max() < 1e-10 and np.abs(zz[:, 6:10] - zk[:, 6:10]).max() < 1e-10
        q = zz[:, 6:10]
        assert np.abs(np.linalg.norm(q, axis=1) - 1).max() < 1e-12


# ----------------------------------------------------------------------------------------------------------------
# contact data (SURVEY.md 8 f4: get_contact_gradients, gradients/contact.jl; data blocks gradients/data.jl:152-192)
# ----------------------------------------------------------------------------------------------------------------
def _perturbed_contact(mech, ci, p, delta):
    import copy
    m2 = copy.deepcopy(mech)
    c = m2.contacts[ci]
    if p == 0:
        c.friction += delta
    elif p == 1:
        c.radius += delta
    else:
        o = np.array(c.origin, dtype=float)
        o[p - 2] += delta
        c.origin = o
    return m2


@pytest.mark.parametrize("name,steps", [("ant", 30), ("quadruped", 40)])
def test_contact_data_jacobian_matches_finite_difference(name, steps):
    """test/data.jl for the contact data: the analytic blocks == central differences of the residual with respect to
    [friction_coefficient, contact_radius, contact_origin] at a fixed solution (contacts active after the roll-in)"""
    mech = dj.get_mechanism(name)
    o = Oracle(mech, capi.solver_options(rtol=1e-10, btol=1e-10))
    u = np.zeros(mech.nu)
    z = _advance(Oracle(mech), mech, mech.z0.copy(), u, steps)
    zn, st, _, sol = o.step(z, u, return_sol=True)
    assert st == 0
    o.set_state(z, u)
    o.set_solution(sol, 0.0)
    D = o.contact_data_jacobian()
    assert np.abs(D).max() > 0.1
    eps = 1e-6
    for ci in range(mech.Ni):
        for p in range(5):
            r = []
            for sgn in (1.0, -1.0):
                o2 = Oracle(_perturbed_contact(mech, ci, p, sgn * eps))
                o2.set_state(z, u)
                o2.set_solution(sol, 0.0)
                r.append(o2.evaluate_rhs(sol, 0.0))
            assert np.abs((r[0] - r[1]) / (2 * eps) - D[:, 5 * ci + p]).max() < 1e-7


def test_contact_gradients_match_finite_difference_of_the_step():
    """get_contact_gradients == d z' / d(contact data) by central differences of the step itself (quadruped standing on
    sticking contacts: a well-conditioned KKT system; at a sliding contact the IFT system of the reference has a condition
    number ~1e10 and its solution is not a usable reference for finite differences)"""
    mech = dj.get_mechanism("quadruped")
    opts = capi.solver_options(rtol=1e-11, btol=1e-11)
    o = Oracle(mech, opts)
    u = np.zeros(mech.nu)
    z = _advance(Oracle(mech), mech, mech.z0.copy(), u, 40)
    zn, _, _, st, _ = o.step_grad(z, u)
    Fc = o.contact_gradients()
    assert st == 0 and np.abs(Fc).max() > 1.0
    eps = 1e-6
    for ci in (0, 3):
        for p in range(5):
            zp, _, _ = Oracle(_perturbed_contact(mech, ci, p, eps), opts).step(z, u)
            zm, _, _ = Oracle(_perturbed_contact(mech, ci, p, -eps), opts).step(z, u)
            fd = (_reduce(zp, zn, mech.Nb) - _reduce(zm, zn, mech.Nb)) / (2 * eps)
            assert np.abs(fd - Fc[:, 5 * ci + p]).max() < 1e-5 * max(1.0, np.abs(Fc).max())
