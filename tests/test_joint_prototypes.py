"""All 16 joint prototypes (src/joints/prototypes.jl:482-499: the (N_lambda_tra, N_lambda_rot) table) with springs and dampers on both
halves, as the reference sweeps them in test/damper.jl (:1-17: a two-body snake per joint type, dampers = 0.3):
oracle: KKT matrix and data Jacobian == finite differences; device kernels (emulation): step, solution vector and IFT gradients == oracle.
"""
import numpy as np
import pytest

import dojo_jl_b200 as dj
from dojo_jl_b200 import capi, quat as Q
from dojo_jl_b200.mechanism import Body, Joint, Mechanism
from oracle.oracle import Oracle

from test_oracle_properties import _perturb_state
from test_translational_joints import _element

PROTOTYPES = {"Fixed": (3, 3), "Prismatic": (2, 3), "Planar": (1, 3), "FixedOrientation": (0, 3), "Revolute": (3, 2), "Cylindrical": (2, 2),
              "PlanarAxis": (1, 2), "FreeRevolute": (0, 2), "Orbital": (3, 1), "PrismaticOrbital": (2, 1), "PlanarOrbital": (1, 1),
              "FreeOrbital": (0, 1), "Spherical": (3, 0), "CylindricalFree": (2, 0), "PlanarFree": (1, 0), "Floating": (0, 0)}


def snake(joint_type, spring=0.2, damper=0.3):
    """two links; link 1 floats, link 2 hangs on it through `joint_type` about / along a skew axis (snake/mechanism.jl with num_bodies = 2)"""
    nt, nr = PROTOTYPES[joint_type]
    bodies = [Body(f"link{i}", 1.0 + 0.2 * i, np.diag([0.08, 0.09, 0.02]) * (1 + 0.3 * i)) for i in range(2)]
    axis = np.array([0.2, 1.0, 0.3])
    j0 = Joint("float", -1, 0, _element(0), _element(0))
    j1 = Joint("joint", 0, 1, _element(nt, axis=axis, spring=spring, damper=damper, offset=0.05 * np.arange(1, 4 - nt)),
               _element(nr, axis=axis, spring=spring, damper=damper, offset=0.1 * np.arange(1, 4 - nr)),
               vertex_parent=np.array([0.0, 0.05, -0.5]), vertex_child=np.array([0.02, 0.0, 0.5]), orientation_offset=Q.rpy_to_quat([0.1, 0.2, -0.1]))
    m = Mechanism(f"snake_{joint_type}", bodies, [j0, j1], [], timestep=0.01, gravity=(0.0, 0.0, -9.81))
    coords = {"float": [0.0, 0.1, 1.0, 0.3, -0.2, 0.1]}
    if j1.input_dimension:
        coords["joint"] = list(0.1 * np.arange(1, j1.input_dimension + 1))
    m.z0 = m.forward_kinematics(coords)
    return m


def _moving_state(m, steps=8):
    o = Oracle(m)
    rng = np.random.default_rng(12)
    z, u = m.z0.copy(), 0.3 * rng.normal(size=m.nu)
    for _ in range(steps):
        z, st, _ = o.step(z, u)
        assert st == 0
    return z, u


@pytest.mark.parametrize("joint_type,inputs", [pytest.param(t, "zero", id=t) for t in PROTOTYPES] +
                         [pytest.param(t, "nonzero", id=f"{t}-inputs") for t in PROTOTYPES])
def test_oracle_blocks_match_finite_differences(joint_type, inputs):
    """KKT matrix and data Jacobian of the oracle == central differences of its residual.  With nonzero inputs the state columns
    carry d(input impulse)/d(x2, q2) of every translational / rotational input, applied between a floating parent and its child."""
    m = snake(joint_type)
    z, u = _moving_state(m)
    o = Oracle(m, capi.solver_options(rtol=1e-9, btol=1e-9))
    u0 = np.zeros(m.nu) if inputs == "zero" else u
    _, _, _, sol = o.step(z, u0, return_sol=True)
    o.set_state(z, u0)
    o.set_solution(sol, 0.0)
    A, _ = o.assemble(0.0)
    D = o.data_jacobian()
    d = 1e-6
    for i in range(m.nres):
        sp, sm = sol.copy(), sol.copy()
        sp[i] += d
        sm[i] -= d
        assert np.abs((o.evaluate_rhs(sp, 0.0) - o.evaluate_rhs(sm, 0.0)) / (2 * d) + A[:, i]).max() < 1e-6
    for i in range(12 * m.Nb):
        o.set_state(_perturb_state(z, i, d), u0)
        rp = o.evaluate_rhs(sol, 0.0)
        o.set_state(_perturb_state(z, i, -d), u0)
        rm = o.evaluate_rhs(sol, 0.0)
        assert np.abs((rp - rm) / (2 * d) - D[:, i]).max() < 2e-6


@pytest.mark.parametrize("joint_type", list(PROTOTYPES))
def test_device_kernels_match_oracle(joint_type):
    from hostemu.harness import HostEmu
    m = snake(joint_type)
    o, em = Oracle(m), HostEmu(m)
    rng = np.random.default_rng(14)
    B = 2
    Z = np.tile(m.z0, (B, 1))
    U = 0.3 * rng.normal(size=(B, m.nu))
    for t in range(12):
        Zn, st, it, sol = em.step(Z, U, slots=2)
        for e in range(B):
            zo, so, io, solo = o.step(Z[e], U[e], return_sol=True)
            assert (st[e], it[e]) == (so, io)
            assert np.abs(Zn[e] - zo).max() < 1e-10 and np.abs(sol[e] - solo).max() < 1e-8
        Z = Zn
    Zn, Fz, Fu, st, it = em.step_grad(Z, U, slots=2, slots_grad=2)
    for e in range(B):
        zo, Fzo, Fuo, so, io = o.step_grad(Z[e], U[e])
        assert (st[e], it[e]) == (so, io)
        assert np.abs(Fz[e] - Fzo).max() < 1e-8 * max(1.0, np.abs(Fzo).max()) and np.abs(Fu[e] - Fuo).max() < 1e-8 * max(1.0, np.abs(Fuo).max())


LIMITED = [("Revolute", "rot"), ("Orbital", "rot"), ("Spherical", "rot"), ("Prismatic", "tra"), ("Planar", "tra"), ("FixedOrientation", "tra"),
           ("Cylindrical", "rot"), ("Cylindrical", "tra")]


@pytest.mark.parametrize("joint_type,half", LIMITED)
def test_limits_on_every_number_of_free_axes(joint_type, half):
    """joints/limits.jl on 1, 2 and 3 limited axes of either half (the device condenses up to three limited axes per joint): step,
    solution vector (slacks and duals in the reference ordering) and gradients against the oracle, with a limit active"""
    from hostemu.harness import HostEmu
    m = snake(joint_type, spring=0.0, damper=0.1)
    j = m.joints[1]
    el = j.rot if half == "rot" else j.tra
    n = el.nfree
    c0 = 0.1 * np.arange(1, j.input_dimension + 1)
    c0 = c0[j.tra.nfree:] if half == "rot" else c0[:j.tra.nfree]
    el.limit_lo, el.limit_hi = c0 - 0.03, c0 + 0.04   # tight box around the initial coordinates: the inputs push into it
    o, em = Oracle(m), HostEmu(m)
    rng = np.random.default_rng(15)
    B = 2
    Z = np.tile(m.z0, (B, 1))
    U = np.zeros((B, m.nu))
    U[:, 6:] = 3.0 * rng.normal(size=(B, m.nu - 6))
    gmax = 0.0
    jo, nb = m.joint_sol_offset(1), 2 * n
    for t in range(25):
        Zn, st, it, sol = em.step(Z, U, slots=2)
        for e in range(B):
            zo, so, io, solo = o.step(Z[e], U[e], return_sol=True)
            assert (st[e], it[e]) == (so, io)
            assert np.abs(Zn[e] - zo).max() < 1e-9 and np.abs(sol[e] - solo).max() < 1e-7
            s0 = jo + (0 if half == "tra" else j.tra.nimpulses)   # [s (nb) | gamma (nb) | eq] inside the limited half
            gmax = max(gmax, solo[s0 + nb: s0 + 2 * nb].max())
        Z = Zn
    assert gmax > 0.05
    Zn, Fz, Fu, st, it = em.step_grad(Z, U, slots=2, slots_grad=2)
    for e in range(B):
        zo, Fzo, Fuo, so, io = o.step_grad(Z[e], U[e])
        assert (st[e], it[e]) == (so, io)
        assert np.abs(Fz[e] - Fzo).max() < 1e-7 * max(1.0, np.abs(Fzo).max()) and np.abs(Fu[e] - Fuo).max() < 1e-7 * max(1.0, np.abs(Fuo).max())
