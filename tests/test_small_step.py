"""The forward kernel specialised for small mechanisms (dojo_step_kernel<false, true, false, SMALL = true>) -- CPU suite on the kernel
emulation (tests/hostemu/small.py).

The specialisation decides from constants what the generic kernel reads from the plan (2 warps per environment, paired line-search
trials, joint pairs, at most 16 nodes per role pass, plan in shared memory); its floating-point operations are the generic kernel's in
the same order.  So, for every mechanism dojo_create hands it, its results must be BIT-IDENTICAL to the generic kernel's: states,
status, Newton iterations and the full solution vector, for single steps, fused rollouts and every thread order of the emulation.
The selection rule (dojo_b200.cu, small_step_ok) must pick it exactly for those mechanisms.  The -m gpu twin is
tests/test_zzzzz_gpu_small_step.py.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import dojo_jl_b200 as dj
from conftest import jittered_states, random_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SWITCHES = ("DOJO_B200_WARPS", "DOJO_B200_NO_JOINT_PAIR", "DOJO_B200_NO_LS_PAIR", "DOJO_B200_NO_LS_ASSIST", "DOJO_B200_SLOTS",
            "DOJO_B200_GLOBAL_PLAN", "DOJO_B200_GENERIC_PLAN", "DOJO_B200_GENERIC_STEP")
# every mechanism of the package that qualifies, and the 16-node boundary shape of tests/test_shape_boundaries.py
QUALIFY = ("ant", "quadruped", "pendulum", "cartpole", "slider", "w16")


def _mech(name):
    """a mechanism of the package, or a synthetic shape of tests/test_shape_boundaries.py"""
    from test_shape_boundaries import SHAPES, shape
    return shape(name) if name in SHAPES else dj.get_mechanism(name)


def _emu(m):
    from hostemu.small import SmallEmu
    return SmallEmu(m)


@pytest.fixture
def clean_env(monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    return monkeypatch


def _start(m, B, seed, rollin=3):
    """B states after `rollin` emulated steps from jittered configurations (contacts closing, bodies in motion) and the next inputs"""
    rng = np.random.default_rng(seed)
    Z = jittered_states(m, B, rng) if m.Nb > 2 else np.tile(m.z0, (B, 1)) + rng.normal(0.0, 1e-3, (B, m.nz)) * (np.arange(m.nz) % 13 >= 10)
    em = _emu(m)
    for _ in range(rollin):
        Z = em.step(Z, random_inputs(m, B, rng, 0.5), slots=2)[0]
    return Z, random_inputs(m, B, rng, 0.5)


# ----------------------------------------------------------------------------------------------------------------
# selection rule
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", QUALIFY)
def test_selected_for_small_mechanisms(name, clean_env):
    em = _emu(_mech(name))
    assert em.small_step_ok(), f"{name} no longer runs the kernel specialised for small mechanisms"
    assert not em.small_step_ok(smem_plan=False), "selected with the plan tables outside shared memory"


@pytest.mark.parametrize("name,env", [
    ("atlas", {}),                                  # 4 warps: more than 16 nodes of a kind
    ("b17", {}), ("c17", {}),                       # 17 bodies / 17 contacts: 4 warps
    ("b17", {"DOJO_B200_WARPS": "2"}),              # 17 nodes in one pass at 2 warps: one-lane fallbacks
    ("chain32", {}),                                # the 32-link chain
    ("raiberthopper", {}), ("block", {}),           # the DJ_ANY_CONTACT compilation / no paired line search
    ("ant", {"DOJO_B200_NO_JOINT_PAIR": "1"}),
    ("ant", {"DOJO_B200_NO_LS_PAIR": "1"}),
    ("ant", {"DOJO_B200_WARPS": "1"}), ("ant", {"DOJO_B200_WARPS": "4"}), ("ant", {"DOJO_B200_WARPS": "8"}),
    ("ant", {"DOJO_B200_GLOBAL_PLAN": "1"}),
    ("ant", {"DOJO_B200_GENERIC_PLAN": "1"}),
    ("ant", {"DOJO_B200_GENERIC_STEP": "1"}),
])
def test_generic_kernel_elsewhere(name, env, clean_env):
    for k, v in env.items():
        clean_env.setenv(k, v)
    em = _emu(_mech(name))
    # GLOBAL_PLAN leaves every table in global memory (dojo_create: plan_smem_mask = 0)
    assert not em.small_step_ok(smem_plan="DOJO_B200_GLOBAL_PLAN" not in env), f"{name} {env}: the specialised kernel would run"


def test_a_qualifying_mechanism_reaches_every_condition(clean_env):
    """the rule's inputs for ant, so that a change of dojo_create's heuristics names the condition that no longer holds"""
    from test_shape_boundaries import _plan_config
    em = _emu(_mech("ant"))
    cfg = _plan_config(em)
    assert em.L.hostemu_warps_per_env(em.h) == 2 and cfg["ls_pair"] == 1 and cfg["jpair"] == 1


# ----------------------------------------------------------------------------------------------------------------
# bit-identity with the generic kernel
# ----------------------------------------------------------------------------------------------------------------
def _same(a, b, what):
    for k, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), f"{what}: output {k} differs (max |diff| {np.max(np.abs(np.asarray(x, float) - np.asarray(y, float)))})"


@pytest.mark.parametrize("name", QUALIFY)
def test_steps_are_bit_identical(name, clean_env):
    m = _mech(name)
    em = _emu(m)
    B = 5
    Z, U = _start(m, B, seed=7)
    for slots, grid in ((1, 1), (2, 2), (4, 1)):  # slots = 4 on one CTA: the drained slots assist the line search of the last one
        gen = em.step(Z, U, slots=slots, grid=grid)
        small = em.step_small(Z, U, slots=slots, grid=grid)
        _same(gen, small, f"{name} slots={slots}")
        assert np.all(gen[1] == 0) or name == "w16", f"{name}: steps did not converge: {gen[1]}"


@pytest.mark.parametrize("name", ("ant", "quadruped", "pendulum"))
def test_fused_rollouts_are_bit_identical(name, clean_env):
    m = _mech(name)
    em = _emu(m)
    B, T = 3, 4
    Z, _ = _start(m, B, seed=11, rollin=1)
    U = np.stack([random_inputs(m, B, np.random.default_rng(100 + t), 0.5) for t in range(T)])
    gen = em.step(Z, U, T=T, slots=2, grid=1, record=True)
    small = em.step_small(Z, U, T=T, slots=2, grid=1, record=True)
    _same(gen, small, f"{name} rollout T={T}")


def test_max_iter_and_line_search_limits_are_bit_identical(clean_env):
    """a solver budget that ends steps :failed, and a line search of one trial per iteration (no paired second trial)"""
    from dojo_jl_b200 import capi
    m = _mech("ant")
    em = _emu(m)
    Z, U = _start(m, 4, seed=5)
    for kw in ({"max_iter": 3}, {"max_ls": 1}, {"max_ls": 3}):
        o = capi.solver_options(**kw)
        _same(em.step(Z, U, opts=o, slots=4), em.step_small(Z, U, opts=o, slots=4), f"ant {kw}")


ORDERS = r"""
import sys, numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests")
import dojo_jl_b200 as dj
from hostemu.small import SmallEmu
from conftest import jittered_states, random_inputs
out = {}
for name in ("ant", "quadruped"):
    m = dj.get_mechanism(name)
    em = SmallEmu(m)
    rng = np.random.default_rng(43)
    Z = jittered_states(m, 4, rng)
    U = random_inputs(m, 4, rng, 0.5)
    for t in range(2):
        Z = em.step(Z, U, slots=2)[0]
    r = em.step_small(Z, U, slots=4)
    f = em.step_small(Z, np.tile(U, (3, 1, 1)), T=3, slots=2, grid=2)
    for k, v in enumerate(r):
        out[f"{name}_step{k}"] = v
    for k, v in enumerate(f):
        out[f"{name}_roll{k}"] = v
    g = em.step(Z, U, slots=4)
    for k, v in enumerate(g):
        out[f"{name}_gen{k}"] = v
np.savez(sys.argv[1], **out)
"""


def _run_order(order, path):
    env = dict(os.environ)
    env.pop("HOSTEMU_ORDER", None)
    for k in SWITCHES:
        env.pop(k, None)
    if order:
        env["HOSTEMU_ORDER"] = order
    r = subprocess.run([sys.executable, "-c", ORDERS % {"root": ROOT}, path], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    if order:
        assert "thread order of a round = " + order in r.stderr
    return np.load(path)


def test_thread_orders_are_bit_identical(tmp_path):
    """the specialised kernel under HOSTEMU_ORDER=reverse|random equals the generic kernel in ascending order (a race in the constant
    warp count, the unrolled reductions or the schedule would show here)"""
    ref = _run_order(None, str(tmp_path / "asc.npz"))
    for name in ("ant", "quadruped"):
        for k in range(4):
            assert np.array_equal(ref[f"{name}_gen{k}"], ref[f"{name}_step{k}"]), (name, k)
    for order in ("reverse", "random"):
        got = _run_order(order, str(tmp_path / (order + ".npz")))
        for k in ref.files:
            assert np.array_equal(ref[k], got[k]), (order, k)
