"""Closed-loop rollouts (dojo_rollout_feedback) -- CPU suite on the kernel emulation.

The closed-loop rollout kernel (dojo_step_kernel<..., FB = true>) evaluates the linear feedback law on the minimal state before every step
and then runs dojo_rollout's step on the input it computed.  So dojo_rollout driven by the returned U_applied must reproduce its trajectory,
final state and status BIT FOR BIT, for every contact model, any number of slots and every thread order of the emulation; the kernel's
minimal state must be the host map's bit for bit, and U_applied / xi the law's.  The -m gpu twin is tests/test_zzzzzzz_gpu_rollout_feedback.py.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import dojo_jl_b200 as dj
from conftest import jittered_states

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ("pendulum", "cartpole", "ant", "quadruped", "raiberthopper", "block_linear")


def _mech(name):
    if name == "block_linear":
        return dj.get_mechanism("block", contact_type="linear")
    return dj.get_mechanism(name)


def _emu(m):
    from hostemu.feedback import FeedbackEmu
    return FeedbackEmu(m)


def _start(m, B, seed):
    """B states in motion: bodies thrown at the ground, jittered joints"""
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
    return Z


def _law(m, B, T, seed, scale=0.3):
    """a per-(step, environment) law with every term: K, K_i [T, B, nu, 2nu], x_ref [T, B, 2nu], u_ref [T, B, nu], xi [B, 2nu]"""
    rng = np.random.default_rng(seed)
    nu = m.nu
    return dict(K=rng.normal(0.0, scale, (T, B, nu, 2 * nu)), K_i=rng.normal(0.0, scale, (T, B, nu, 2 * nu)),
                x_ref=rng.normal(0.0, 0.1, (T, B, 2 * nu)), u_ref=rng.normal(0.0, 0.3, (T, B, nu)), xi=rng.normal(0.0, 0.05, (B, 2 * nu)))


def _same(got, ref, what):
    for k, (g, r) in enumerate(zip(got, ref)):
        if g is None and r is None:
            continue
        assert g.shape == r.shape, (what, k, g.shape, r.shape)
        assert np.array_equal(g, r, equal_nan=True), f"{what}: output {k} differs (max |diff| {np.nanmax(np.abs(g - r))})"


def _check_open_loop(em, Z0, out, slots, what):
    """dojo_rollout driven by U_applied reproduces Z_traj, Z_final and status_any bit for bit"""
    Zf, st, traj, Ua = out[:4]
    T = Ua.shape[0]
    Zo, sto, _, _, trajo = em.step(Z0, Ua, T=T, slots=slots, grid=2, record=True)
    _same((traj, Zf, st), (trajo, Zo, sto), what)


@pytest.mark.parametrize("name", CASES)
def test_equals_open_loop_rollout(name):
    m = _mech(name)
    em = _emu(m)
    B, T = 3, 4
    Z0 = _start(m, B, seed=21)
    out = em.rollout_feedback(Z0, T, **_law(m, B, T, seed=22))
    assert np.isfinite(out[3]).all()
    _check_open_loop(em, Z0, out, 2, name)
    # without U_applied the kernel writes u_t to its scratch: the same trajectory
    _same(em.rollout_feedback(Z0, T, applied=False, **_law(m, B, T, seed=22))[:3], out[:3], name + " (no U_applied)")


@pytest.mark.parametrize("slots", (1, 4))
@pytest.mark.parametrize("name", ("ant", "block_linear"))
def test_slots(name, slots):
    m = _mech(name)
    em = _emu(m)
    B, T = 5, 3
    Z0 = _start(m, B, seed=23)
    law = _law(m, B, T, seed=24)
    out = em.rollout_feedback(Z0, T, slots=slots, grid=2, **law)
    _check_open_loop(em, Z0, out, slots, f"{name} slots={slots}")
    _same(out, em.rollout_feedback(Z0, T, slots=2, grid=2, **law), f"{name} slots={slots} against 2 slots")


@pytest.mark.parametrize("name", ("pendulum", "ant", "block_linear"))
def test_law(name):
    """x_t is the host map's on the state before step t, bit for bit; U_applied and xi are the law evaluated in numpy to 1e-14 of the sum of
    the magnitudes of its terms"""
    from hostcheck.harness import HostCheck
    m = _mech(name)
    em, hc = _emu(m), HostCheck(m)
    B, T = 3, 4
    Z0 = _start(m, B, seed=25)
    law = _law(m, B, T, seed=26)
    Zf, st, traj, Ua, xi, x_last = em.rollout_feedback(Z0, T, **law)
    before = np.concatenate([Z0[None], traj[:-1]])  # the state each step starts from
    X = hc.maximal_to_minimal(before.reshape(T * B, -1)).reshape(T, B, -1)
    assert np.array_equal(x_last, X[-1]), np.abs(x_last - X[-1]).max()
    for t0 in range(1, T):  # x_t of an earlier step: the last step of a shorter run from the same start
        assert np.array_equal(em.rollout_feedback(Z0, t0, **{k: (v[:t0] if k != "xi" else v) for k, v in law.items()})[5], X[t0 - 1]), t0
    h, z = m.timestep, law["xi"].copy()
    for t in range(T):
        dx = X[t] - law["x_ref"][t]
        z = z + h * dx
        terms = [law["u_ref"][t], -np.einsum("bik,bk->bi", law["K"][t], dx), -np.einsum("bik,bk->bi", law["K_i"][t], z)]
        mag = np.abs(law["u_ref"][t]) + np.einsum("bik,bk->bi", np.abs(law["K"][t]), np.abs(dx)) + np.einsum("bik,bk->bi", np.abs(law["K_i"][t]), np.abs(z))
        err = np.abs(Ua[t] - sum(terms))
        assert (err <= 1e-14 * mag).all(), (t, (err / mag).max())
    assert (np.abs(xi - z) <= 1e-14 * (np.abs(law["xi"]) + h * np.abs(X - law["x_ref"]).sum(axis=0))).all()


def test_broadcasting():
    """one law for all, per environment, per step and per pair, and terms left out, each against the explicitly tiled [T, B] arrays"""
    m = _mech("cartpole")
    em = _emu(m)
    B, T, nu = 3, 4, m.nu
    Z0 = _start(m, B, seed=27)
    law = _law(m, B, T, seed=28)

    def tiled(v, k):
        shape = {"K": (nu, 2 * nu), "K_i": (nu, 2 * nu), "x_ref": (2 * nu,), "u_ref": (nu,)}[k]
        n = v.ndim - len(shape)
        v = v.reshape(((1, 1), (1, B), v.shape[:2])[n] + shape)
        return np.broadcast_to(v, (T, B) + shape)

    forms = {"shared": lambda v: v[0, 0], "per env": lambda v: v[0], "per step": lambda v: v[:, :1], "per pair": lambda v: v}
    for kf, f in forms.items():
        for mix in (False, True):
            # mix: the other arrays in the other forms, so that the common (steps, envs) comes from different arrays
            keys = ("K", "K_i", "x_ref", "u_ref")
            fs = [f] + ([forms[o] for o in forms if o != kf] if mix else [f] * 3)
            given = {k: g(law[k]) for k, g in zip(keys, fs)}
            got = em.rollout_feedback(Z0, T, xi=law["xi"], **given)
            ref = em.rollout_feedback(Z0, T, xi=law["xi"], **{k: tiled(v, k) for k, v in given.items()})
            _same(got, ref, f"{kf} mix={mix}")
    # absent terms: the same as zeros
    got = em.rollout_feedback(Z0, T, K=law["K"])
    ref = em.rollout_feedback(Z0, T, K=law["K"], x_ref=np.zeros(2 * nu), u_ref=np.zeros(nu))
    _same(got, ref, "absent x_ref / u_ref")
    assert got[4] is None


def test_continuation():
    """T1 + T2 steps with Z_final and xi passed on equal one run of T1 + T2 steps bit for bit"""
    m = _mech("ant")
    em = _emu(m)
    B, T1, T2 = 3, 2, 3
    Z0 = _start(m, B, seed=29)
    law = _law(m, B, T1 + T2, seed=30)
    one = em.rollout_feedback(Z0, T1 + T2, **law)
    a = em.rollout_feedback(Z0, T1, **{k: (v[:T1] if k != "xi" else v) for k, v in law.items()})
    b = em.rollout_feedback(a[0], T2, **{k: (v[T1:] if k != "xi" else a[4]) for k, v in law.items()})
    _same((b[0], np.maximum(a[1], b[1]), np.concatenate([a[2], b[2]]), np.concatenate([a[3], b[3]]), b[4]), one[:5], "continuation")


PID = dict(Kp=25.0, Ki=50.0, Kd=5.0, goal=np.pi / 2, steps=500)


def _pid_law():
    p = PID
    return dict(K=np.array([[p["Kp"], p["Kd"]]]), K_i=np.array([[p["Ki"], 0.0]]), x_ref=np.array([p["goal"], 0.0]))


def test_pendulum_pid_against_oracle():
    """examples/control/pendulum_pid.jl (Kp = 25, Ki = 50, Kd = 5, goal pi/2, 5 s from rest at angle 0): the emulated closed loop agrees
    with a host loop of oracle steps under the same law to 1e-8 over all 500 steps, and ends within 1e-3 rad of the goal"""
    from oracle.oracle import Oracle
    m = _mech("pendulum")
    o = Oracle(m)
    em = _emu(m)
    z0 = o.minimal_to_maximal(np.zeros(2))
    Zf, st, traj, Ua, xi, _ = em.rollout_feedback(z0[None], PID["steps"], **_pid_law())
    assert st[0] == 0
    # the reference: summed_error += (goal - x[1]) h; u = Kp (goal - x[1]) + Ki summed_error + Kd (0 - x[2])
    z, s, ref = z0, 0.0, []
    for k in range(PID["steps"]):
        x = o.maximal_to_minimal(z)
        s += (PID["goal"] - x[0]) * m.timestep
        u = PID["Kp"] * (PID["goal"] - x[0]) + PID["Ki"] * s + PID["Kd"] * (0.0 - x[1])
        r = o.step(z, np.array([u]))
        z = r[0] if isinstance(r, tuple) else r
        ref.append(z)
    ref = np.array(ref)
    assert np.abs(traj[:, 0] - ref).max() < 1e-8, np.abs(traj[:, 0] - ref).max()
    assert abs(xi[0, 0] + s) < 1e-8
    theta = o.maximal_to_minimal(Zf[0])[0]
    assert abs(theta - PID["goal"]) < 1e-3, theta


ORDERS = r"""
import sys, numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests")
from test_rollout_feedback import _mech, _emu, _start, _law
out = {}
for name in ("ant", "block_linear"):
    m = _mech(name)
    for k, v in enumerate(_emu(m).rollout_feedback(_start(m, 4, seed=31), 3, slots=2, grid=2, **_law(m, 4, 3, seed=32))):
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
    """HOSTEMU_ORDER=reverse|random: a race between the map, the integral, the law and the prologue that reads u_t would show here"""
    ref = _run_order(None, str(tmp_path / "asc.npz"))
    for order in ("reverse", "random"):
        got = _run_order(order, str(tmp_path / (order + ".npz")))
        for k in ref.files:
            assert np.array_equal(ref[k], got[k], equal_nan=True), (order, k)


def test_feedback_arrays_refuses_bad_shapes():
    from dojo_jl_b200.solver import feedback_arrays
    nu, B, T = 2, 3, 4
    K = np.ones((nu, 2 * nu))
    steps, envs, Kc, xr, ur, Ki = feedback_arrays(T, B, nu, K, x_ref=np.zeros((B, 2 * nu)))
    assert (steps, envs, Kc.shape, xr.shape, ur, Ki) == (1, B, (1, B, 2 * nu, nu), (1, B, 2 * nu), None, None)
    for bad in (np.ones((nu, nu)), np.ones((B + 1, nu, 2 * nu)), np.ones((T + 1, 1, nu, 2 * nu)), np.ones((T, 2, nu, 2 * nu))):
        with pytest.raises(ValueError):
            feedback_arrays(T, B, nu, bad)


def test_ctypes_mirror_matches_the_c_header(tmp_path):
    """DojoFeedback: size and field offsets as the C compiler lays them out == the ctypes mirror in dojo.jl_b200/capi.py"""
    from dojo_jl_b200 import capi
    st = capi.DojoFeedback
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "dojo_b200.h")}"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(DojoFeedback));']
    lines += [f'  printf("{f} %zu\\n", offsetof(DojoFeedback, {f}));' for f, _ in st._fields_]
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-o", str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(out["size"]) == C.sizeof(st)
    for f, _ in st._fields_:
        assert int(out[f]) == getattr(st, f).offset, f
