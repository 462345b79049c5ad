"""Reverse mode through a fused rollout (dojo_rollout_tape + dojo_rollout_vjp) -- CPU suite on the kernel emulation.

The tape is the recording rollout of dojo_rollout_grad without the gradient kernel, so its trajectory, status and iterations must equal
rollout_grad's bit for bit.  The adjoint kernel (dojo_step_kernel<true, ..., VJP = true>) solves one transposed system per step instead of
12Nb + nu columns, so its gZ0 / gU agree with the contraction of rollout_grad's Jacobians up to rounding, and must not depend on the slot
count, the thread order or the batch.  The -m gpu twin is tests/test_zzzzzzzzzz_gpu_rollout_vjp.py.
"""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import dojo_jl_b200 as dj
from conftest import jittered_states, random_inputs
from dojo_jl_b200 import capi, solver
from dojo_jl_b200.autograd import attitude_map, from_attitude, to_attitude

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ("pendulum", "cartpole", "ant", "quadruped", "raiberthopper", "block_linear")


def _mech(name):
    if name == "block_linear":
        return dj.get_mechanism("block", contact_type="linear")
    return dj.get_mechanism(name)


def _emu(m):
    from hostemu.vjp import VjpEmu
    return VjpEmu(m)


def _start(m, B, T, seed, scale=0.5):
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
        Z = np.tile(m.z0, (B, 1)) + rng.normal(0.0, 1e-1, (B, m.nz)) * (np.arange(m.nz) % 13 >= 10)
    U = np.stack([random_inputs(m, B, rng, scale) for _ in range(T)])
    return Z, U


def _slots_grad(m):
    return 1 if m.Nb > 13 else 2


def contract(Fz, Fu, gZ):
    """lambda_T = gZ[T]; gU[t] = Fu[t]' lambda_{t+1}; lambda_t = Fz[t]' lambda_{t+1} + gZ[t] -- and the same recursion in absolute values"""
    T = Fz.shape[0]
    lam, lamA = gZ[T].copy(), np.abs(gZ[T])
    gU, gUa = np.zeros(Fu.shape[:2] + Fu.shape[3:]), np.zeros(Fu.shape[:2] + Fu.shape[3:])
    for t in range(T - 1, -1, -1):
        gU[t], gUa[t] = np.einsum("bij,bi->bj", Fu[t], lam), np.einsum("bij,bi->bj", np.abs(Fu[t]), lamA)
        lam, lamA = np.einsum("bij,bi->bj", Fz[t], lam) + gZ[t], np.einsum("bij,bi->bj", np.abs(Fz[t]), lamA) + np.abs(gZ[t])
    return lam, gU, lamA, gUa


# Tolerance relative to the bound of assert_close.  Ant is the exception: once its feet touch down and its joints reach their limits, the
# column solves and the transposed solve disagree by far more than the absolute contraction accounts for -- up to 3.6e-7 of the bound in
# ONE step (tests/hostemu, seed 21, steps 3 to 6; 2e-15 at step 0, before contact).  Both are solves against the same factor of a KKT
# system whose condensed contact and limit rows carry gamma / s ratios of a converged interior point, so neither is exact to that
# level; pendulum, cartpole, quadruped, raiberthopper and the linear-contact block agree to 1e-13 of the bound or better.
TOL = {"ant": 1e-6}


def assert_close(got, ref, bound, what, tol=1e-11):
    """|got - ref| <= tol * (bound + max of bound over the environment's vector): the entrywise bound of the absolute contraction, plus
    its largest entry in the same vector.  A small entry of Fu or Fz is the residue of a cancellation inside the KKT solve; the transposed
    solve takes it in another order, so its rounding scales with the vector, not with the entry."""
    scale = bound + bound.max(axis=-1, keepdims=True)
    err = np.abs(got - ref)
    ok = err <= tol * scale
    assert ok.all(), f"{what}: worst {np.max(err / np.maximum(scale, 1e-300)):.2e} of the bound at {np.argwhere(~ok)[:4].tolist()}"


@pytest.mark.parametrize("name", CASES)
def test_matches_jacobian_contraction(name):
    """gZ0 / gU against the numpy contraction of the emulated rollout_grad Jacobians, random cotangents on every slab; a solver budget
    that ends some pairs :failed (their Jacobians are those of the final iterate, and so is the adjoint)"""
    m = _mech(name)
    em = _emu(m)
    B, T = 3, 8 if m.Nb > 2 else 12
    Z0, U = _start(m, B, T, seed=21)
    opts = capi.solver_options(max_iter=8) if name in ("ant", "quadruped") else None
    traj, Fz, Fu, st, it = em.rollout_grad(Z0, U, T, opts, slots=2, slots_grad=_slots_grad(m), grid=2)
    traj2, tape, st2, it2 = em.rollout_tape(Z0, U, T, opts, slots=2, grid=2)
    assert np.array_equal(traj, traj2) and np.array_equal(st, st2) and np.array_equal(it, it2)
    if opts is not None:
        assert (st == 1).any(), f"no pair ended :failed: {st}"
    gZ = np.random.default_rng(22).normal(size=(T + 1, B, 12 * m.Nb))
    gZ0, gU, vst = em.rollout_vjp(traj2, U, tape, gZ, slots_grad=_slots_grad(m), grid=2)
    assert (vst == 0).all(), vst
    lam, gUr, lamA, gUa = contract(Fz, Fu, gZ)
    assert_close(gZ0, lam, lamA, f"{name} gZ0", TOL.get(name, 1e-11))
    assert_close(gU, gUr, gUa, f"{name} gU", TOL.get(name, 1e-11))


@pytest.mark.parametrize("name", ("pendulum", "ant", "block_linear"))
def test_tape_matches_recording_rollout(name):
    """the tape's trajectory, status and iterations: rollout_grad's and, for the trajectory and the worst status, dojo_rollout's"""
    m = _mech(name)
    em = _emu(m)
    B, T = 4, 5
    Z0, U = _start(m, B, T, seed=23)
    traj, _, _, st, it = em.rollout_grad(Z0, U, T, slots=2, slots_grad=_slots_grad(m), grid=2)
    traj2, tape, st2, it2 = em.rollout_tape(Z0, U, T, slots=2, grid=2)
    assert np.array_equal(traj, traj2) and np.array_equal(st, st2) and np.array_equal(it, it2)
    Zf, st_any, _, _, tr = em.step(Z0, U, T=T, slots=2, record=True)
    assert np.array_equal(traj2[1:], tr) and np.array_equal(traj2[-1], Zf) and np.array_equal(st2.max(axis=0), st_any)


def _vjp_case(m, B, T, seed):
    em = _emu(m)
    Z0, U = _start(m, B, T, seed)
    traj, tape, _, _ = em.rollout_tape(Z0, U, T, slots=2, grid=2)
    gZ = np.random.default_rng(seed + 1).normal(size=(T + 1, B, 12 * m.Nb))
    return em, traj, U, tape, gZ


@pytest.mark.parametrize("name", ("ant", "block_linear"))
def test_slots_and_batch_are_bit_identical(name):
    """1 and 4 slots per CTA, 1 and 3 CTAs; environment e of a batch of 8 equals the same environment run alone"""
    m = _mech(name)
    B, T = 8, 3
    em, traj, U, tape, gZ = _vjp_case(m, B, T, 24)
    ref = em.rollout_vjp(traj, U, tape, gZ, slots_grad=1, grid=1)
    for slots, grid in ((4, 1), (2, 3)):
        got = em.rollout_vjp(traj, U, tape, gZ, slots_grad=slots, grid=grid)
        for g, r in zip(got, ref):
            assert np.array_equal(g, r), (name, slots, grid)
    got = em.rollout_vjp(traj, U, tape, gZ, slots_grad=1, grid=1, smem_plan=False)
    for g, r in zip(got, ref):
        assert np.array_equal(g, r), (name, "plan in global memory")
    for e in (0, 5):
        one = em.rollout_vjp(traj[:, e:e + 1].copy(), U[:, e:e + 1].copy(), tape[:, e:e + 1].copy(), gZ[:, e:e + 1].copy(), slots_grad=2)
        assert np.array_equal(one[0][0], ref[0][e]) and np.array_equal(one[1][:, 0], ref[1][:, e]) and one[2][0] == ref[2][e], (name, e)


ORDERS = r"""
import sys, numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests")
from test_rollout_vjp import _mech, _vjp_case
out = {}
for name in ("ant", "block_linear"):
    em, traj, U, tape, gZ = _vjp_case(_mech(name), 4, 3, 25)
    for k, v in enumerate(em.rollout_vjp(traj, U, tape, gZ, slots_grad=2, grid=2)):
        out[f"{name}_{k}"] = v
    out[f"{name}_tape"] = tape
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
    """HOSTEMU_ORDER=reverse|random: a race between the lanes of the transposed sweeps, the scratch folds or the update of lambda would
    show here"""
    ref = _run_order(None, str(tmp_path / "asc.npz"))
    for order in ("reverse", "random"):
        got = _run_order(order, str(tmp_path / (order + ".npz")))
        for k in ref.files:
            assert np.array_equal(ref[k], got[k], equal_nan=True), (order, k)


def test_zero_cotangents_give_exact_zeros():
    m = _mech("ant")
    em, traj, U, tape, gZ = _vjp_case(m, 2, 3, 26)
    gZ0, gU, st = em.rollout_vjp(traj, U, tape, np.zeros_like(gZ), slots_grad=2)
    assert (st == 0).all() and np.array_equal(gZ0, np.zeros_like(gZ0)) and np.array_equal(gU, np.zeros_like(gU))


def test_nonfinite_factorisation_is_confined_to_its_environment():
    """a NaN in the tape of environment 1 at step 1: status 3 and NaN outputs for that environment; the others bit for bit as without it"""
    m = _mech("ant")
    em, traj, U, tape, gZ = _vjp_case(m, 3, 3, 27)
    ref = em.rollout_vjp(traj, U, tape, gZ, slots_grad=2, grid=2)
    bad = tape.copy()
    bad[1, 1, :] = np.nan
    gZ0, gU, st = em.rollout_vjp(traj, U, bad, gZ, slots_grad=2, grid=2)
    assert st.tolist() == [0, 3, 0]
    assert np.isnan(gZ0[1]).all() and np.isnan(gU[:, 1]).all()
    for e in (0, 2):
        assert np.array_equal(gZ0[e], ref[0][e]) and np.array_equal(gU[:, e], ref[1][:, e])


def test_without_input_cotangent_buffer():
    """gU is nullable: gZ0 is the same without it"""
    m = _mech("raiberthopper")
    em, traj, U, tape, gZ = _vjp_case(m, 2, 3, 28)
    ref = em.rollout_vjp(traj, U, tape, gZ, slots_grad=2)
    gZ0, gU, st = em.rollout_vjp(traj, U, tape, gZ, slots_grad=2, with_gU=False)
    assert gU is None and np.array_equal(gZ0, ref[0]) and np.array_equal(st, ref[2])


def _rollout_loss(em, Z0, U, c, d, opts):
    Zf, _, _, _, tr = em.step(Z0, U, opts, T=U.shape[0], slots=1, record=True)
    return float(c @ Zf[0] + sum(d @ z[0] for z in tr[:-1]) + d @ Z0[0])


def _perturb(m, z, k, eps):
    """z moved by eps along coordinate k of the gradients' packing [x, v, phi, w] per body; attitudes along q (x) (1, eps e)"""
    z = z.copy()
    b, i = divmod(k, 12)
    o = 13 * b
    if i < 6:
        z[o + i] += eps
    elif i >= 9:
        z[o + i + 1] += eps
    else:
        q = z[o + 6:o + 10].copy()
        dq = np.zeros(3)
        dq[i - 6] = eps
        qn = q + attitude_map(q) @ dq  # q (x) (1, eps e), exactly (the product is linear in its second factor)
        z[o + 6:o + 10] = qn / np.linalg.norm(qn)
    return z


@pytest.mark.parametrize("name", ("pendulum", "cartpole"))
def test_central_differences(name):
    """the scalar loss c' z_T + sum_{t<T} d' z_t, solved at rtol = btol = 1e-11: gU and gZ0 against central differences"""
    m = _mech(name)
    em = _emu(m)
    T = 6
    Z0, U = _start(m, 1, T, seed=29)
    opts = capi.solver_options(rtol=1e-11, btol=1e-11, max_iter=100)
    rng = np.random.default_rng(30)
    c, d = rng.normal(size=m.nz), rng.normal(size=m.nz)
    traj, tape, st, _ = em.rollout_tape(Z0, U, T, opts)
    assert (st == 0).all()
    gZ = np.stack([to_attitude(traj[t], np.broadcast_to(c if t == T else d, traj[t].shape)) for t in range(T + 1)])
    gZ0, gU, vst = em.rollout_vjp(traj, U, tape, gZ)
    assert vst[0] == 0
    eps = 1e-6
    fd_u = np.zeros_like(gU)
    for t in range(T):
        for j in range(m.nu):
            Up, Um = U.copy(), U.copy()
            Up[t, 0, j] += eps
            Um[t, 0, j] -= eps
            fd_u[t, 0, j] = (_rollout_loss(em, Z0, Up, c, d, opts) - _rollout_loss(em, Z0, Um, c, d, opts)) / (2 * eps)
    fd_z = np.zeros(12 * m.Nb)
    for k in range(12 * m.Nb):
        fd_z[k] = (_rollout_loss(em, _perturb(m, Z0[0], k, eps)[None], U, c, d, opts) -
                   _rollout_loss(em, _perturb(m, Z0[0], k, -eps)[None], U, c, d, opts)) / (2 * eps)
    scale = max(1.0, np.abs(fd_z).max(), np.abs(fd_u).max())
    assert np.abs(gU - fd_u).max() < 1e-6 * scale, (np.abs(gU - fd_u).max(), scale)
    assert np.abs(gZ0[0] - fd_z).max() < 1e-6 * scale, (np.abs(gZ0[0] - fd_z).max(), scale)


def test_attitude_maps():
    """G(q) = d(q (x) (1, d))/dd by finite differences; phibar = G' qbar is the derivative of a loss along q (x) (1, d); G(q) phibar is
    tangent to the unit sphere (q' G(q) = 0); both maps leave the other coordinates alone"""
    rng = np.random.default_rng(31)
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    G = attitude_map(q)

    def qmul(a, b):
        return np.array([a[0] * b[0] - a[1:] @ b[1:], *(a[0] * b[1:] + b[0] * a[1:] + np.cross(a[1:], b[1:]))])
    h = 1e-7
    fd = np.stack([(qmul(q, np.r_[1.0, h * e]) - qmul(q, np.r_[1.0, -h * e])) / (2 * h) for e in np.eye(3)], -1)
    assert np.abs(fd - G).max() < 1e-8
    assert np.abs(q @ G).max() < 1e-15
    W = rng.normal(size=(4, 4))
    loss = lambda p: np.sin(p @ W @ p)  # noqa: E731
    qbar = np.cos(q @ W @ q) * (W + W.T) @ q
    dphi = np.array([(loss(qmul(q, np.r_[1.0, h * e])) - loss(qmul(q, np.r_[1.0, -h * e]))) / (2 * h) for e in np.eye(3)])
    z = np.concatenate([rng.normal(size=6), q, rng.normal(size=3)])
    gz = np.concatenate([rng.normal(size=6), qbar, rng.normal(size=3)])
    g12 = to_attitude(z, gz)
    assert np.abs(g12[6:9] - dphi).max() < 1e-7
    assert np.array_equal(g12[:6], gz[:6]) and np.array_equal(g12[9:], gz[10:])
    back = from_attitude(z, g12)
    assert np.array_equal(back[:6], gz[:6]) and np.array_equal(back[10:], gz[10:]) and abs(q @ back[6:10]) < 1e-15
    # batched, several bodies: the same per body
    Z = np.stack([np.concatenate([z, z]), np.concatenate([z, z])])
    GZ = np.stack([np.concatenate([gz, 2 * gz]), np.concatenate([gz, gz])])
    out = to_attitude(Z, GZ)
    assert out.shape == (2, 24) and np.allclose(out[0, 12:], 2 * g12, rtol=0, atol=1e-15) and np.allclose(out[1, :12], g12, rtol=0, atol=1e-15)


def _prototype_params(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dojo_b200.h")).read(), flags=re.S)
    m = re.search(r"\b%s\s*\(([^)]*)\)" % name, text)
    assert m, name
    return [p.strip() for p in m.group(1).split(",")]


@pytest.mark.parametrize("name", ("dojo_rollout_tape", "dojo_rollout_tape_async", "dojo_rollout_vjp", "dojo_rollout_vjp_async"))
def test_ctypes_prototypes_match_header(name):
    """argument count and integer / pointer kinds of the ctypes prototypes against include/dojo_b200.h"""
    import __graft_entry__ as ge
    ge.build()
    L = solver.load_library()
    fn = getattr(L, name)
    params = _prototype_params(name)
    assert len(fn.argtypes) == len(params), (name, params)
    for a, p in zip(fn.argtypes, params):
        if "*" in p:
            assert a in (C.c_void_p, C.POINTER(capi.DojoSolverOptions)), (name, p, a)
        else:
            assert a is C.c_int, (name, p, a)
    assert fn.restype is C.c_int


def test_refusals_without_handle():
    """a null handle is refused before anything else is read"""
    import __graft_entry__ as ge
    ge.build()
    L = solver.load_library()
    assert L.dojo_rollout_tape(None, None, 1, 1, None, None, None, None, None, None) == -1
    assert L.dojo_rollout_vjp(None, 1, 1, None, None, None, None, None, None, None) == -1
