"""Trajectory Jacobians of a fused rollout (dojo_rollout_grad, dojo_rollout_minimal_gradients) -- CPU suite on the kernel emulation.

The recording rollout (dojo_step_kernel<..., REC = true>) runs the Newton loop of dojo_rollout and keeps, per (environment, step) pair
t * B + e, the final solution, the status and the iterations; the unchanged gradient kernel then runs over the B * T pairs.  So its
results must be BIT-IDENTICAL to T sequential dojo_step_grad calls (states, per-step status and iterations, Fz, Fu), and its trajectory
and status to dojo_rollout's, for every contact model, both compilations, any number of slots and every thread order of the emulation.
The -m gpu twin is tests/test_zzzzzz_gpu_rollout_grad.py.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import dojo_jl_b200 as dj
from conftest import jittered_states, random_inputs
from dojo_jl_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ("pendulum", "ant", "quadruped", "raiberthopper", "block_linear")


def _mech(name):
    if name == "block_linear":
        return dj.get_mechanism("block", contact_type="linear")
    return dj.get_mechanism(name)


def _emu(m):
    from hostemu.rollout_grad import RolloutGradEmu
    return RolloutGradEmu(m)


def _start(m, B, T, seed):
    """B states in motion (bodies thrown at the ground, jittered joints) and T steps of inputs"""
    rng = np.random.default_rng(seed)
    if m.name == "block":
        Z = np.tile(m.z0, (B, 1))
        Z[:, 2] += rng.uniform(-0.9, 0.0, B)
        Z[:, 3:6] = rng.normal(size=(B, 3)) * [1.0, 1.0, 0.3]
        Z[:, 10:13] = rng.normal(size=(B, 3))
    elif m.Nb > 2:
        Z = jittered_states(m, B, rng)
    else:
        Z = np.tile(m.z0, (B, 1)) + rng.normal(0.0, 1e-3, (B, m.nz)) * (np.arange(m.nz) % 13 >= 10)
    U = np.stack([random_inputs(m, B, rng, 0.5) for _ in range(T)])
    return Z, U


def _slots_grad(m):
    return 1 if m.Nb > 13 else 2


def _sequential(em, m, Z0, U, opts=None):
    """T dojo_step_grad calls, each from the state the previous one returned"""
    Z, out = Z0, []
    for t in range(U.shape[0]):
        r = em.step_grad(Z, U[t], opts, slots=2, slots_grad=_slots_grad(m))
        out.append(r)
        Z = r[0]
    traj = np.stack([Z0] + [r[0] for r in out])
    return traj, np.stack([r[1] for r in out]), np.stack([r[2] for r in out]), np.stack([r[3] for r in out]), np.stack([r[4] for r in out])


def _same(got, ref, what):
    for k, (g, r) in enumerate(zip(got, ref)):
        assert g.shape == r.shape, (what, k, g.shape, r.shape)
        assert np.array_equal(g, r, equal_nan=True), f"{what}: output {k} differs (max |diff| {np.nanmax(np.abs(g - r))})"


@pytest.mark.parametrize("name", CASES)
def test_equals_sequential_step_grad(name):
    m = _mech(name)
    em = _emu(m)
    B, T = 3, 4
    Z0, U = _start(m, B, T, seed=11)
    got = em.rollout_grad(Z0, U, T, slots=2, slots_grad=_slots_grad(m), grid=2)
    _same(got, _sequential(em, m, Z0, U), name)
    # the trajectory and the status of dojo_rollout
    Zf, st_any, _, _, traj = em.step(Z0, U, T=T, slots=2, record=True)
    assert np.array_equal(got[0][1:], traj) and np.array_equal(got[0][-1], Zf)
    assert np.array_equal(got[3].max(axis=0), st_any)


@pytest.mark.parametrize("slots", (1, 4))
@pytest.mark.parametrize("name", ("ant", "block_linear"))
def test_slots(name, slots):
    m = _mech(name)
    em = _emu(m)
    B, T = 5, 3
    Z0, U = _start(m, B, T, seed=12)
    got = em.rollout_grad(Z0, U, T, slots=slots, slots_grad=1, grid=2)
    _same(got, _sequential(em, m, Z0, U), f"{name} slots={slots}")


def test_failed_middle_step():
    """a solver budget that ends some steps :failed: every pair carries its own step's status and iterations, and the steps after a
    failed one are what dojo_step_grad computes from the state the failed step returned"""
    m = _mech("ant")
    em = _emu(m)
    B, T = 4, 5
    Z0, U = _start(m, B, T, seed=13)
    U[2] *= 8.0  # a hard kick in the middle of the trajectory
    opts = capi.solver_options(max_iter=10)
    got = em.rollout_grad(Z0, U, T, opts, slots=2, slots_grad=_slots_grad(m), grid=2)
    ref = _sequential(em, m, Z0, U, opts)
    _same(got, ref, "ant max_iter=10")
    st = got[3]
    assert (st == 1).any() and (st == 0).any(), st
    assert ((st[1:-1] == 1).any()), f"no middle step ended :failed: {st}"


def test_minimal_equals_per_step_composition():
    """minimal coordinates: the map-Jacobian kernel between slabs t and t + 1 of the rollout, the same kernel applied to the states and
    Jacobians of T sequential dojo_step_grad calls; and the chained minimal-coordinate steps within rounding of the coordinate maps"""
    from hostemu.adapter import EmuStepper
    from hostemu.rollout_grad import rollout_minimal_gradients
    for name in ("pendulum", "ant"):
        m = _mech(name)
        s, em = EmuStepper(m, 8), _emu(m)
        B, T = 3, 3
        Z0, U = _start(m, B, T, seed=14)
        X0 = s.maximal_to_minimal(Z0)
        Xt, Gx, Gu, st, it = rollout_minimal_gradients(em, s.hc, X0, U, T, slots_grad=_slots_grad(m))
        traj, Fz, Fu, st2, it2 = _sequential(em, m, s.minimal_to_maximal(X0), U)
        assert np.array_equal(st, st2) and np.array_equal(it, it2)
        for t in range(T):
            gx, gu = s.hc.minimal_gradients(traj[t], traj[t + 1], Fz[t], Fu[t])
            assert np.array_equal(Gx[t], gx) and np.array_equal(Gu[t], gu), (name, t)
        assert np.array_equal(Xt, s.maximal_to_minimal(traj.reshape((T + 1) * B, -1)).reshape(T + 1, B, -1))
        # the first step is one get_minimal_gradients! call from X0; a chain of such calls re-enters maximal coordinates at every step,
        # so from the second step on it starts the solver from a state that differs in the last bits and agrees to its tolerance
        Xn, gx, gu, st0, it0 = s.minimal_gradients(X0, U[0])
        _same((Xn, gx, gu, st0, it0), (Xt[1], Gx[0], Gu[0], st[0], it[0]), name)
        for t in range(1, T):
            Xn = s.minimal_gradients(Xn, U[t])[0]
            assert np.allclose(Xn, Xt[t + 1], rtol=1e-5, atol=1e-6), (name, t, np.abs(Xn - Xt[t + 1]).max())


ORDERS = r"""
import sys, numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests")
from test_rollout_grad import _mech, _emu, _start, _slots_grad
out = {}
for name in ("ant", "block_linear"):
    m = _mech(name)
    Z0, U = _start(m, 4, 3, seed=15)
    for k, v in enumerate(_emu(m).rollout_grad(Z0, U, 3, slots=2, slots_grad=_slots_grad(m), grid=2)):
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
    """HOSTEMU_ORDER=reverse|random: a race between the recording epilogue, the publication of a pair and its gradient would show here"""
    ref = _run_order(None, str(tmp_path / "asc.npz"))
    for order in ("reverse", "random"):
        got = _run_order(order, str(tmp_path / (order + ".npz")))
        for k in ref.files:
            assert np.array_equal(ref[k], got[k], equal_nan=True), (order, k)
