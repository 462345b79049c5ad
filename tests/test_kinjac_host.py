"""Jacobians of the minimal <-> maximal maps and get_minimal_gradients! (SURVEY.md 8 f1) -- CPU tests.

 * the oracle's literal restatement (gradients/state.jl:9-56, :136-217; joints/minimal.jl:206-400) is pinned by the
   reference's own property test (test/minimal.jl:378-560): analytic Jacobians == finite differences of the maps times the
   attitude Jacobian, and M N = I;
 * the DEVICE code (dojo.jl_b200/csrc/dojo_kinjac.cuh, closed forms in attitude coordinates) is compiled for the host by
   tests/hostcheck and compared with the oracle entry by entry.  The same functions run on the GPU in
   tests/test_zz_gpu_kinjac.py through the C-ABI.
"""
import numpy as np
import pytest

import dojo_jl_b200 as dj
from dojo_jl_b200 import capi
from oracle.oracle import Oracle

from hostcheck.harness import HostCheck
from test_oracle_properties import _perturb_state, _random_minimal, _reduce

MECHS = ["pendulum", "ant", "quadruped", "atlas"]


def _states(mech, o, rng, n):
    """on-manifold maximal states with velocities, incl. one with every joint coordinate exactly zero (theta = 0 branches)"""
    out = []
    for k in range(n):
        x = _random_minimal(mech, rng)
        if k == n - 1:
            x[:] = 0.0
        out.append((x, o.minimal_to_maximal(x)))
    return out


@pytest.mark.parametrize("name", MECHS)
def test_oracle_map_jacobians_match_finite_differences(name):
    """test/minimal.jl:378-560: M_a == M_fd (1e-8 there with ForwardDiff; central differences here), N_a == N_fd, M N = I."""
    mech = dj.get_mechanism(name)
    o = Oracle(mech)
    rng = np.random.default_rng(11)
    x, z = _states(mech, o, rng, 1)[0]
    M = o.maximal_to_minimal_jacobian(z)
    N = o.minimal_to_maximal_jacobian(z)
    assert M.shape == (2 * mech.nu, 12 * mech.Nb) and N.shape == (12 * mech.Nb, 2 * mech.nu)
    eps = 1e-6
    Mfd = np.stack([(o.maximal_to_minimal(_perturb_state(z, i, eps)) - o.maximal_to_minimal(_perturb_state(z, i, -eps))) / (2 * eps)
                    for i in range(12 * mech.Nb)], axis=1)
    assert np.abs(M - Mfd).max() < 2e-7
    cols = []
    for i in range(2 * mech.nu):
        xp, xm = x.copy(), x.copy()
        xp[i] += eps
        xm[i] -= eps
        cols.append((_reduce(o.minimal_to_maximal(xp), z, mech.Nb) - _reduce(o.minimal_to_maximal(xm), z, mech.Nb)) / (2 * eps))
    assert np.abs(N - np.stack(cols, axis=1)).max() < 2e-7
    assert np.abs(M @ N - np.eye(2 * mech.nu)).max() < 1e-11


def test_reference_body_order_quirk():
    """gradients/state.jl:170-178 chains the partials in mechanism.bodies order.  With parents listed before children that
    IS the derivative; otherwise (atlas here, URDF order) rows of late parents are missing -- the reference disables its own
    check for such models (test/minimal.jl:527, :560).  The product chains root -> leaves."""
    rng = np.random.default_rng(2)
    for name in MECHS:
        mech = dj.get_mechanism(name)
        o = Oracle(mech)
        z = o.minimal_to_maximal(_random_minimal(mech, rng))
        parents_first = all(j.parent < j.child for j in mech.joints)
        diff = np.abs(o.minimal_to_maximal_jacobian(z) - o.minimal_to_maximal_jacobian(z, body_order_literal=True)).max()
        assert (diff == 0.0) if parents_first else (diff > 1e-3), (name, parents_first, diff)


@pytest.mark.parametrize("name", MECHS)
def test_device_code_on_host_matches_oracle(name):
    mech = dj.get_mechanism(name)
    o, hc = Oracle(mech), HostCheck(mech)
    rng = np.random.default_rng(7)
    st = _states(mech, o, rng, 4)
    X = np.stack([s[0] for s in st])
    Z = np.stack([s[1] for s in st])
    # the maps themselves (dojo_kin.cuh)
    assert np.abs(hc.minimal_to_maximal(X) - Z).max() < 1e-12
    assert np.abs(hc.maximal_to_minimal(Z) - X).max() < 1e-10
    # constraint violation at solver-tolerance level (unit quaternions): still the same numbers
    Zv = Z.copy().reshape(len(st), mech.Nb, 13)
    Zv[:, :, 0:6] += 1e-5 * rng.normal(size=Zv[:, :, 0:6].shape)
    Zv[:, :, 10:13] += 1e-5 * rng.normal(size=Zv[:, :, 10:13].shape)
    Zv[:, :, 6:10] += 1e-5 * rng.normal(size=Zv[:, :, 6:10].shape)
    Zv[:, :, 6:10] /= np.linalg.norm(Zv[:, :, 6:10], axis=2, keepdims=True)
    Zv = Zv.reshape(len(st), -1)
    for Zs in (Z, Zv):
        Mh, Nh = hc.maximal_to_minimal_jacobian(Zs), hc.minimal_to_maximal_jacobian(Zs)
        for e in range(len(st)):
            M, N = o.maximal_to_minimal_jacobian(Zs[e]), o.minimal_to_maximal_jacobian(Zs[e])
            assert np.abs(Mh[e] - M).max() < 1e-10 * max(1.0, np.abs(M).max())
            assert np.abs(Nh[e] - N).max() < 1e-10 * max(1.0, np.abs(N).max())


@pytest.mark.parametrize("name", ["pendulum", "ant", "quadruped"])
def test_minimal_gradients_device_code_on_host_matches_oracle(name):
    mech = dj.get_mechanism(name)
    o, hc = Oracle(mech), HostCheck(mech)
    rng = np.random.default_rng(9)
    for _ in range(2):
        x = _random_minimal(mech, rng, 0.1, 0.2)
        if name != "pendulum":
            x[2] += 0.4  # lift the floating base off the ground
        u = rng.uniform(-1, 1, mech.nu)
        xn, Gx, Gu, st, _ = o.minimal_gradients(x, u)
        z = o.minimal_to_maximal(x)
        zn, Fz, Fu, _, _ = o.step_grad(z, u)
        Gxh, Guh = hc.minimal_gradients(z, zn, Fz[None], Fu[None])
        assert st == 0
        assert np.abs(Gxh[0] - Gx).max() < 1e-10 * max(1.0, np.abs(Gx).max())
        assert np.abs(Guh[0] - Gu).max() < 1e-10 * max(1.0, np.abs(Gu).max())


def test_minimal_gradients_match_finite_differences_of_the_minimal_step():
    """get_minimal_gradients! is the derivative of step_minimal_coordinates! (a tight solve and no active contact, so the step is
    smooth: the pendulum, and ant / quadruped / raiberthopper lifted 3 m with random inputs on every actuated joint, where the inputs'
    configuration derivative (SURVEY Q17) belongs to Fz.  In minimal coordinates it shows for raiberthopper's prismatic leg, whose
    input torque has a lever arm that moves along the joint; a revolute joint's input torque lies on its own axis.)"""
    for name in ("pendulum", "ant", "quadruped", "raiberthopper"):
        _minimal_gradients_match_finite_differences(name)


def _minimal_gradients_match_finite_differences(name):
    from conftest import random_inputs
    mech = dj.get_mechanism(name)
    opts = capi.solver_options(rtol=1e-11, btol=1e-11)
    o = Oracle(mech, opts)
    if name == "pendulum":
        x = np.array([0.7, -0.4])
        u = np.array([0.3])
    else:
        rng = np.random.default_rng(4)
        x = _random_minimal(mech, rng, 0.2, 0.5)
        x[2] += 3.0  # floating base height
        u = random_inputs(mech, 1, rng)[0]

    def f(x_, u_):
        zn, st, it = o.step(o.minimal_to_maximal(x_), u_)
        assert st == 0
        return o.maximal_to_minimal(zn), it

    xn, Gx, Gu, st, it0 = o.minimal_gradients(x, u)
    assert st == 0 and np.abs(xn - f(x, u)[0]).max() < 1e-12
    eps, n, checked = 1e-6, 2 * mech.nu, 0
    for i in range(n + mech.nu):
        d = np.zeros(n + mech.nu)
        d[i] = eps
        (fp, ip), (fm, im) = f(x + d[:n], u + d[n:]), f(x - d[:n], u - d[n:])
        if ip != it0 or im != it0:
            continue  # a different Newton-iteration count changes the (tolerance-level) solver error: FD noise / eps
        G = Gx[:, i] if i < n else Gu[:, i - n]
        assert np.abs((fp - fm) / (2 * eps) - G).max() < 1e-6 * max(1.0, np.abs(G).max()), (name, i, np.abs((fp - fm) / (2 * eps) - G).max())
        checked += 1
    assert checked >= (n + mech.nu) // 2, name
