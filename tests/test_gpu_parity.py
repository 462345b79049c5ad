"""GPU parity tests (run with -m gpu on an H100): the CUDA path, called through the C-ABI, against the CPU
oracle on identical seeded inputs.

Bar (BASELINE.json north_star: fp64 tolerance, identical contact modes):
  * same status for every environment;
  * environments whose Newton-iteration count equals the oracle's:  |z_next - z_oracle|_inf <= 1e-6 (typically 1e-12; rounding is amplified by ill-conditioned contact solves) and an identical
    contact-mode bitmap (gamma_1 > s_1 per contact);
  * iteration counts may differ for a small fraction of environments (a rounding-level flip of a line-search /
    convergence comparison, SURVEY.md §7 hard part 2); those must still agree to solver tolerance.
"""
import numpy as np
import pytest

import dojo_jl_b200 as dj
from dojo_jl_b200 import capi
from conftest import jittered_states, random_inputs

pytestmark = pytest.mark.gpu

TOL_SAME_PATH = 1e-6    # every same-iteration environment (3.3e-7 measured once in 3072 ant environments in hard contact) ...
TOL_SAME_Q99 = 1e-9     # ... and 99 % of them (SURVEY.md 8c asks for 1e-9; the median is ~1e-13)
# Environments that take a different number of Newton iterations on the two paths: a rounding-level flip of the convergence
# comparison (rvio < rtol && bvio < btol) makes one path stop one iterate earlier / later on the SAME central path.  Consecutive
# iterates near convergence differ by up to ~1e-2 with the reference defaults (rtol 1e-6, btol 1e-4; e.g. ant at rest: iterate 6 vs 7
# = 8.1e-3, iterate 7 vs 8 = 7.5e-4), so a fixed bound on |z_gpu - z_oracle| says nothing there.  Instead the oracle is re-run with
# EXACTLY the device's iteration count (Oracle.step_forced, a test hook that skips the convergence test) and must then agree like a
# same-iteration environment (TOL_SAME_PATH).  What that does not explain -- a flipped line-search comparison earlier in the solve,
# i.e. a different path -- is counted separately, must stay below TOL_SOLVER and below MAX_PATH_FLIPS of the environment-steps.
TOL_SOLVER = 2e-2
MAX_PATH_FLIPS = 0.002


def _contact_modes(mech, sol):
    """gamma_1 > s_1 per contact: a contact's entry is [s(N/2); gamma(N/2)] for every model, normal component first"""
    idx = np.array([mech.contact_sol_offset(c) for c in range(mech.Ni)], dtype=int)
    half = np.array([c.dim // 2 for c in mech.contacts], dtype=int)
    return sol[:, idx + half] > sol[:, idx]


def _compare_rollout(name, B, T, seed, scale, opts=None, max_mismatch=0.01, tol_same=TOL_SAME_PATH, tol_all=TOL_SOLVER, tol_median=None):
    """`name`: a mechanism name or a Mechanism.  tol_median: optional bound on the median same-iteration error."""
    from dojo_jl_b200.solver import BatchedStepper
    from oracle.oracle import Oracle
    mech = dj.get_mechanism(name) if isinstance(name, str) else name
    name = mech.name
    rng = np.random.default_rng(seed)
    Z = jittered_states(mech, B, rng) if mech.Nb > 1 else np.tile(mech.z0, (B, 1))
    stepper = BatchedStepper(mech, B)
    oracle = Oracle(mech, opts)
    total = mismatched = path_flips = 0
    same_errs, conv_errs, problems, forced_errs = [], [], [], []
    for t in range(T):
        U = random_inputs(mech, B, rng, scale)
        Zg, sg, ig, solg = stepper.step(Z, U, opts=opts, return_sol=True)
        Zo = np.empty_like(Z)
        so, io = np.zeros(B, np.int32), np.zeros(B, np.int32)
        solo = np.empty((B, mech.nres))
        for e in range(B):
            Zo[e], so[e], io[e], solo[e] = oracle.step(Z[e], U[e], return_sol=True)
        # an environment that runs out of Newton iterations on one path (:failed) while the other converges on its last
        # iterations is a tolerance-edge event (the two paths stagnate around the tolerance for dozens of iterations); it is counted in
        # the mismatch budget, everything else must agree
        edge = (sg != so) & (np.maximum(ig, io) >= 45)
        if not ((sg == so) | edge).all():
            problems.append(f"{name} step {t}: status differs")
        conv = (so == 0) & (sg == 0)  # :failed environments end on an arbitrary unconverged iterate
        same = (ig == io) & conv
        err = np.abs(Zg - Zo).max(axis=1)
        if err[same].max(initial=0.0) > tol_same:
            problems.append(f"{name} step {t}: same-iteration error {err[same].max()} > {tol_same}")
        same_errs.append(err[same])
        conv_errs.append(err[conv])
        for e in np.nonzero(conv & (ig != io))[0]:  # the oracle's iterate after exactly the device's number of iterations
            zf, _, _ = oracle.step_forced(Z[e], U[e], int(ig[e]))
            ef = float(np.abs(Zg[e] - zf).max())
            forced_errs.append(ef)
            if ef > tol_same:  # not a flip of the convergence test: a different path
                path_flips += 1
                if err[e] > tol_all:
                    problems.append(f"{name} step {t}: environment {e} took {ig[e]} / {io[e]} iterations and differs by {err[e]} > {tol_all} "
                                    f"({ef} from the oracle's iterate {ig[e]})")
        if mech.Ni and not (_contact_modes(mech, solg)[same] == _contact_modes(mech, solo)[same]).all():
            problems.append(f"{name} step {t}: contact-mode bitmap differs")
        total += B
        mismatched += int((conv & (ig != io)).sum()) + int(edge.sum())
        Z = Zo
    same_errs, conv_errs = np.concatenate(same_errs), np.concatenate(conv_errs)
    _record_stats(name, {"B": B, "T": T, "env_steps": total, "iteration_mismatches": mismatched, "max_err_same_iters": float(same_errs.max()),
                         "q99_err_same_iters": float(np.quantile(same_errs, 0.99)), "median_err_same_iters": float(np.median(same_errs)),
                         "max_err_converged": float(conv_errs.max()), "path_flips": path_flips,
                         "max_err_vs_oracle_iterate_of_same_count": float(max(forced_errs, default=0.0)), "problems": problems[:6]})
    assert not problems, problems[:6]
    assert mismatched <= max_mismatch * total, f"{name}: {mismatched}/{total} environments took a different iteration count"
    assert path_flips <= max(1, MAX_PATH_FLIPS * total), f"{name}: {path_flips}/{total} environments left the oracle's path"
    assert np.quantile(same_errs, 0.99) <= TOL_SAME_Q99, f"{name}: 99 % quantile of the same-iteration error {np.quantile(same_errs, 0.99)}"
    if tol_median is not None:
        assert np.median(same_errs) <= tol_median, f"{name}: median same-iteration error {np.median(same_errs)}"
    return mismatched, total


def _record_stats(name, d):
    """measured parity statistics next to the verdict of the test (captured output: shown on failure, or with pytest -s)"""
    import json
    print("parity_stats " + json.dumps({"test": name, **d}))


def test_pendulum_1000_steps():
    """BASELINE config C0: pendulum, 1 env, 1000 steps."""
    from dojo_jl_b200.solver import BatchedStepper
    from oracle.oracle import Oracle
    mech = dj.get_mechanism("pendulum")
    stepper, oracle = BatchedStepper(mech, 1), Oracle(mech)
    zg = zo = mech.z0.copy()
    for _ in range(1000):
        zg = stepper.step(zg[None], np.zeros((1, 1)))[0][0]
        zo, _, _ = oracle.step(zo, np.zeros(1))
    assert np.abs(zg - zo).max() < 1e-9


def test_rollout_matches_stepwise():
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism("ant")
    rng = np.random.default_rng(3)
    B, T = 16, 6
    Z0 = jittered_states(mech, B, rng)
    U = np.stack([random_inputs(mech, B, rng) for _ in range(T)])
    stepper = BatchedStepper(mech, B)
    Zf, st, traj = stepper.rollout(Z0, U, T, record=True)
    Z = Z0
    for t in range(T):
        Z, s, _ = stepper.step(Z, U[t])
        assert np.array_equal(traj[t], Z)
    assert np.array_equal(Zf, Z)


@pytest.mark.parametrize("name,B,T,scale", [("ant", 96, 25, 1.0), ("quadruped", 64, 30, 2.0), ("atlas", 48, 20, 5.0)])
def test_step_parity(name, B, T, scale):
    _compare_rollout(name, B, T, seed=7, scale=scale)


def test_step_parity_tight_tolerances():
    """rtol = btol = 1e-10 (round 1 stalled below ~1e-8: both sides of every joint limit were condensed through 1 / s; the kept limit
    dual now lives in the joint's node, dojo_plan.h joint_nq): the CUDA path converges wherever the oracle does -- identical status
    for EVERY environment -- and all converged environments agree to 1e-6 whatever their iteration counts (the reference's own
    conservation tests run at 1e-12, test/momentum.jl:154-218).  Same case on the CPU emulation: tests/test_tight_tolerances.py."""
    from dojo_jl_b200.solver import BatchedStepper
    from oracle.oracle import step_batch_threads
    mech = dj.get_mechanism("ant")
    rng = np.random.default_rng(29)
    B = 96
    Z = jittered_states(mech, B, rng)
    stepper = BatchedStepper(mech, B)
    for _ in range(14):
        Z, _, _ = stepper.step(Z, random_inputs(mech, B, rng, 1.0))
    for tol in (1e-10, 1e-12):
        opts = capi.solver_options(rtol=tol, btol=tol)
        U = random_inputs(mech, B, rng, 1.0)
        Zg, sg, ig = stepper.step(Z, U, opts=opts)
        Zo, so, io = step_batch_threads(mech, Z, U, opts, 8)
        conv = (so == 0) & (sg == 0)
        assert conv.sum() >= B // 2
        if tol == 1e-10:
            assert np.array_equal(sg, so), (tol, np.where(sg != so)[0], ig[sg != so], io[sg != so])
        else:  # at 1e-12 both paths sit on their rounding floor: a few environments may end on different sides of the tolerance
            assert (sg != so).sum() <= max(2, B // 20), (tol, (sg != so).sum())
        err = np.abs(Zg - Zo)[conv].max(axis=1)  # ill-conditioned contact solves amplify rounding: 1.1e-6 seen on one environment
        assert err.max() < 1e-5 and np.quantile(err, 0.9) < 1e-7 and np.median(err) < 1e-10, (err.max(), np.quantile(err, 0.9), np.median(err))


def test_two_handles_share_kernels():
    """Handles of different mechanisms share the kernel symbols (the dynamic shared-memory attribute belongs to the function, not to
    the handle): a small mechanism created after a large one must not break the large one's launches, in either order."""
    from dojo_jl_b200.solver import BatchedStepper
    ant, pend = dj.get_mechanism("ant"), dj.get_mechanism("pendulum")
    rng = np.random.default_rng(47)
    Za = jittered_states(ant, 8, rng)
    Ua = random_inputs(ant, 8, rng)
    s_ant = BatchedStepper(ant, 8)
    ref = s_ant.step(Za, Ua)
    s_pend = BatchedStepper(pend, 4)                      # created later, needs a few KB only
    zp = s_pend.step(np.tile(pend.z0, (4, 1)), np.zeros((4, 1)))[0]
    again = s_ant.step(Za, Ua)                            # the large handle still launches
    assert all(np.array_equal(a, b) for a, b in zip(ref, again)) and np.isfinite(zp).all()
    s_atlas = BatchedStepper(dj.get_mechanism("atlas"), 4)  # larger than both
    atlas = dj.get_mechanism("atlas")
    za = s_atlas.step(np.tile(atlas.z0, (4, 1)), np.zeros((4, atlas.nu)))[0]
    assert np.isfinite(za).all()
    assert all(np.array_equal(a, b) for a, b in zip(ref, s_ant.step(Za, Ua)))
    g1 = s_ant.step_grad(Za, Ua)
    s_pend.step_grad(np.tile(pend.z0, (4, 1)), np.zeros((4, 1)))
    g2 = s_ant.step_grad(Za, Ua)
    assert all(np.array_equal(a, b) for a, b in zip(g1, g2))


def test_calls_on_different_streams_are_ordered():
    """One call in flight per handle (include/dojo_b200.h): async calls issued on different streams are ordered by the library, so
    two back-to-back steps on two streams give the results of the same steps issued on one stream."""
    import torch
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism("ant")
    rng = np.random.default_rng(53)
    B = 600
    Z = torch.from_numpy(jittered_states(mech, 32, rng)[rng.integers(0, 32, B)]).cuda()
    U = torch.from_numpy(random_inputs(mech, B, rng)).cuda()
    st = BatchedStepper(mech, B)
    Z1, Z2 = torch.empty_like(Z), torch.empty_like(Z)
    s0 = torch.cuda.current_stream()
    st.step_device(Z.data_ptr(), U.data_ptr(), Z1.data_ptr(), B, stream=s0.cuda_stream)
    st.step_device(Z1.data_ptr(), U.data_ptr(), Z2.data_ptr(), B, stream=s0.cuda_stream)
    torch.cuda.synchronize()
    ref1, ref2 = Z1.clone(), Z2.clone()
    Z1.zero_(); Z2.zero_()
    torch.cuda.synchronize()
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    st.step_device(Z.data_ptr(), U.data_ptr(), Z1.data_ptr(), B, stream=sa.cuda_stream)
    st.step_device(Z1.data_ptr(), U.data_ptr(), Z2.data_ptr(), B, stream=sb.cuda_stream)  # consumes Z1 and the handle's work queue
    torch.cuda.synchronize()
    assert torch.equal(Z1, ref1) and torch.equal(Z2, ref2)


def test_q1_literal_return_flag():
    """step! returns a double-advanced configuration (SURVEY.md Q1); flag bit0 reproduces it."""
    from dojo_jl_b200.solver import BatchedStepper, DOJO_FLAG_Q1_LITERAL_RETURN
    from oracle.oracle import Oracle
    mech = dj.get_mechanism("ant")
    z, u = mech.z0.copy(), np.zeros(mech.nu)
    zg = BatchedStepper(mech, 1).step(z[None], u[None], flags=DOJO_FLAG_Q1_LITERAL_RETURN)[0][0]
    zo, _, _ = Oracle(mech).step(z, u, flags=1)
    assert np.abs(zg - zo).max() < 1e-10
    zt, _, _ = Oracle(mech).step(z, u)
    assert np.abs(zo - zt).max() > 1e-4  # the literal return differs from the true next state


def test_external_force():
    from dojo_jl_b200.solver import BatchedStepper
    from oracle.oracle import Oracle
    mech = dj.get_mechanism("ant")
    rng = np.random.default_rng(5)
    B = 8
    Z = jittered_states(mech, B, rng)
    U = random_inputs(mech, B, rng)
    F = rng.normal(0, 1.0, (B, 6 * mech.Nb))
    Zg, sg, _ = BatchedStepper(mech, B).step(Z, U, fext=F)
    o = Oracle(mech)
    for e in range(B):
        zo, so, _ = o.step(Z[e], U[e], fext=np.ascontiguousarray(F[e]))
        assert np.abs(Zg[e] - zo).max() < 1e-8


def test_full_size_invariants():
    """BASELINE config C1 size (ant, B = 4096): size-independent properties -- unit quaternions, finite output,
    determinism (bit-identical repeat), batch-permutation equivariance."""
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism("ant")
    rng = np.random.default_rng(9)
    B = 4096
    Z = jittered_states(mech, 64, rng)[rng.integers(0, 64, B)]
    Z[:, 2] += rng.uniform(-0.05, 0.2, B)
    U = random_inputs(mech, B, rng)
    stepper = BatchedStepper(mech, B)
    Z1, s1, i1 = stepper.step(Z, U)
    Z2, s2, i2 = stepper.step(Z, U)
    assert np.array_equal(Z1, Z2) and np.array_equal(i1, i2)
    assert np.isfinite(Z1).all() and (s1 == 0).mean() > 0.99
    q = Z1.reshape(B, mech.Nb, 13)[:, :, 6:10]
    assert np.abs(np.linalg.norm(q, axis=2) - 1).max() < 1e-12
    perm = rng.permutation(B)
    Z3, _, _ = stepper.step(Z[perm], U[perm])
    assert np.array_equal(Z3, Z1[perm])


@pytest.mark.parametrize("name,T,scale", [("pendulum", 3, 1.0), ("ant", 20, 1.0), ("quadruped", 25, 1.0), ("atlas", 10, 2.0)])
def test_gradient_parity(name, T, scale):
    """dojo_step_grad (IFT gradients from the retained block-LDU factor, condensed system) vs the oracle's
    get_maximal_gradients restatement (dense `solmat \\ datamat`, gradients/state.jl:99).
    Tolerance, relative to the largest entry: median <= 1e-7 (typically 1e-10), 90 % of the environments <= 1e-4, all
    <= 1e-2.  Contact-rich steps are ill-conditioned -- the oracle's own dense-vs-LDU solves differ by up to 1e-6 there and
    a few environments per batch reach 1e-5 .. 1e-4 between the two factorisation orders."""
    from dojo_jl_b200.solver import BatchedStepper
    from oracle.oracle import Oracle
    mech = dj.get_mechanism(name)
    rng = np.random.default_rng(21)
    B = 12
    Z = jittered_states(mech, B, rng) if mech.Nb > 1 else np.tile(mech.z0, (B, 1))
    stepper, oracle = BatchedStepper(mech, B), Oracle(mech)
    for _ in range(T):
        Z, _, _ = stepper.step(Z, random_inputs(mech, B, rng, scale))
    U = random_inputs(mech, B, rng, scale)
    Zn, Fz, Fu, sg, ig = stepper.step_grad(Z, U)
    Zf, sf, _ = stepper.step(Z, U)
    assert np.array_equal(Zn, Zf)  # the gradient kernel takes the same forward step
    errs = []
    for e in range(B):
        zo, Fzo, Fuo, so, io = oracle.step_grad(Z[e], U[e])
        if so != 0 or sg[e] != 0 or io != ig[e]:
            continue
        scale_z, scale_u = max(1.0, np.abs(Fzo).max()), max(1.0, np.abs(Fuo).max())
        errs.append(max(np.abs(Fz[e] - Fzo).max() / scale_z, np.abs(Fu[e] - Fuo).max() / scale_u))
    errs = np.array(errs)
    assert len(errs) >= B // 2
    assert np.median(errs) < 1e-7 and np.quantile(errs, 0.9) < 1e-4 and errs.max() < 1e-2, errs


def test_batch_size_independence():
    """An environment's result does not depend on the batch it is stepped in (slot / CTA assignment, queue order):
    odd batch sizes (not a multiple of the four slots of a CTA, fewer environments than slots) reproduce the rows of a
    large batch bit for bit."""
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism("ant")
    rng = np.random.default_rng(17)
    B = 601
    Z = jittered_states(mech, 32, rng)[rng.integers(0, 32, B)]
    U = random_inputs(mech, B, rng)
    stepper = BatchedStepper(mech, B)
    Zf, sf, itf = stepper.step(Z, U)
    for b in (1, 3, 5, 149):
        Zb, sb, itb = stepper.step(Z[:b], U[:b])
        assert np.array_equal(Zb, Zf[:b]) and np.array_equal(itb, itf[:b]) and np.array_equal(sb, sf[:b])


def test_pinned_host_buffers():
    """Page-locked caller buffers are copied from / to directly; same results as the staged (pageable) path."""
    import torch
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism("quadruped")
    rng = np.random.default_rng(19)
    B = 64
    Z = jittered_states(mech, B, rng)
    U = random_inputs(mech, B, rng)
    stepper = BatchedStepper(mech, B)
    Zn, st, it = stepper.step(Z, U)
    pin = lambda shape, dt: torch.empty(shape, dtype=dt, pin_memory=True).numpy()
    Zp, Up, Znp = pin(Z.shape, torch.float64), pin(U.shape, torch.float64), pin(Z.shape, torch.float64)
    stp, itp = pin((B,), torch.int32), pin((B,), torch.int32)
    Zp[:], Up[:] = Z, U
    stepper.step(Zp, Up, out=(Znp, stp, itp))
    assert np.array_equal(Znp, Zn) and np.array_equal(stp, st) and np.array_equal(itp, it)


@pytest.mark.parametrize("name", ["pendulum", "quadruped"])
def test_rollout_trajectory(name):
    """dojo_rollout (all steps fused in one launch) records the same trajectory as T single steps."""
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism(name)
    rng = np.random.default_rng(23)
    B, T = 7, 9
    Z0 = jittered_states(mech, B, rng) if mech.Nb > 1 else np.tile(mech.z0, (B, 1))
    U = np.stack([random_inputs(mech, B, rng) for _ in range(T)])
    stepper = BatchedStepper(mech, B)
    Zf, st, traj = stepper.rollout(Z0, U, T, record=True)
    Zf2, st2 = stepper.rollout(Z0, U, T)
    Z, worst = Z0, np.zeros(B, np.int32)
    for t in range(T):
        Z, s, _ = stepper.step(Z, U[t])
        worst = np.maximum(worst, s)
        assert np.array_equal(traj[t], Z)
    assert np.array_equal(Zf, Z) and np.array_equal(Zf2, Z) and np.array_equal(st, worst) and np.array_equal(st2, worst)


# ----------------------------------------------------------------------------------------------------------------
# minimal <-> maximal coordinate maps and step_minimal_coordinates! (SURVEY.md 8 f1)
# ----------------------------------------------------------------------------------------------------------------
def _random_minimal_batch(mech, B, rng):
    X = np.zeros((B, 2 * mech.nu))
    off = 0
    for j in mech.joints:
        n = j.input_dimension
        X[:, 2 * off:2 * off + n] = rng.uniform(-0.3, 0.3, (B, n))
        X[:, 2 * off + n:2 * off + 2 * n] = rng.normal(0.0, 0.5, (B, n))
        off += n
    return X


@pytest.mark.parametrize("name", ["pendulum", "ant", "quadruped", "atlas"])
def test_minimal_maximal_maps(name):
    """dojo_minimal_to_maximal / dojo_maximal_to_minimal vs the oracle's restatement of mechanism/state.jl:9-66, and the
    round trip on the device."""
    from dojo_jl_b200.solver import BatchedStepper
    from oracle.oracle import Oracle
    mech = dj.get_mechanism(name)
    rng = np.random.default_rng(31)
    B = 37
    X = _random_minimal_batch(mech, B, rng)
    stepper, o = BatchedStepper(mech, B), Oracle(mech)
    assert stepper.nmin == 2 * mech.nu
    Z = stepper.minimal_to_maximal(X)
    Zo = np.stack([o.minimal_to_maximal(X[e]) for e in range(B)])
    assert np.abs(Z - Zo).max() < 1e-11
    Xr = stepper.maximal_to_minimal(Z)
    Xo = np.stack([o.maximal_to_minimal(Zo[e]) for e in range(B)])
    assert np.abs(Xr - Xo).max() < 1e-9 and np.abs(Xr - X).max() < 1e-9


@pytest.mark.parametrize("name", ["ant", "quadruped"])
def test_step_minimal_coordinates(name):
    """dojo_step_minimal == maximal_to_minimal(step!(minimal_to_maximal(x), u)) (simulation/step.jl:42-61): bit-identical to the
    composition of the three device calls, and equal to the oracle's composition where the iteration counts agree."""
    from dojo_jl_b200.solver import BatchedStepper
    from oracle.oracle import Oracle
    mech = dj.get_mechanism(name)
    rng = np.random.default_rng(37)
    B = 24
    X = _random_minimal_batch(mech, B, rng)
    off = 0
    for j in mech.joints:  # lift the floating base so that the feet start near the ground, not inside it
        if j.nimpulses == 0:
            X[:, 2 * off + 2] += 0.6
        off += j.input_dimension
    U = random_inputs(mech, B, rng)
    stepper, o = BatchedStepper(mech, B), Oracle(mech)
    Xn, st, it = stepper.step_minimal(X, U)
    Z = stepper.minimal_to_maximal(X)
    Zn, st2, it2 = stepper.step(Z, U)
    assert np.array_equal(Xn, stepper.maximal_to_minimal(Zn)) and np.array_equal(st, st2) and np.array_equal(it, it2)
    for e in range(B):
        zo, so, io = o.step(o.minimal_to_maximal(X[e]), U[e])
        if so == 0 and st[e] == 0 and io == it[e]:
            assert np.abs(Xn[e] - o.maximal_to_minimal(zo)).max() < 1e-6
    # the reference's literal return value (step! advances the configuration a second time, SURVEY.md Q1) in minimal coordinates:
    # dojo_step_minimal_flags(DOJO_FLAG_Q1_LITERAL_RETURN) == maximal_to_minimal(step(..., flags = Q1))
    from dojo_jl_b200.solver import DOJO_FLAG_Q1_LITERAL_RETURN
    Xl, stl, itl = stepper.step_minimal(X, U, flags=DOJO_FLAG_Q1_LITERAL_RETURN)
    Zl, _, _ = stepper.step(Z, U, flags=DOJO_FLAG_Q1_LITERAL_RETURN)
    assert np.array_equal(Xl, stepper.maximal_to_minimal(Zl)) and np.array_equal(stl, st) and np.array_equal(itl, it)
    assert np.abs(Xl - Xn).max() > 1e-6  # it IS a different state
    for e in range(B):
        zo, so, io = o.step(o.minimal_to_maximal(X[e]), U[e], flags=DOJO_FLAG_Q1_LITERAL_RETURN)
        if so == 0 and st[e] == 0 and io == it[e]:
            assert np.abs(Xl[e] - o.maximal_to_minimal(zo)).max() < 1e-6


def test_full_size_invariants_quadruped():
    """BASELINE config C2 size (quadruped, B = 8192, forward + gradients): size-independent properties -- unit quaternions,
    determinism, permutation equivariance of states AND gradients, gradient launch leaves the forward result untouched."""
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism("quadruped")
    rng = np.random.default_rng(41)
    B = 8192
    Z = jittered_states(mech, 64, rng)[rng.integers(0, 64, B)]
    Z[:, 2] += rng.uniform(0.0, 0.1, B)
    U = random_inputs(mech, B, rng)
    stepper = BatchedStepper(mech, B)
    Z1, s1, i1 = stepper.step(Z, U)
    Z2, s2, i2 = stepper.step(Z, U)
    assert np.array_equal(Z1, Z2) and np.array_equal(i1, i2) and np.isfinite(Z1).all()
    q = Z1.reshape(B, mech.Nb, 13)[:, :, 6:10]
    assert np.abs(np.linalg.norm(q, axis=2) - 1).max() < 1e-12
    n = 512  # gradients on a slice (215 KB per environment)
    perm = rng.permutation(n)
    Zg, Fz, Fu, sg, ig = stepper.step_grad(Z[:n], U[:n])
    Zp, Fzp, Fup, _, _ = stepper.step_grad(Z[:n][perm], U[:n][perm])
    assert np.array_equal(Zg, Z1[:n]) and np.array_equal(ig, i1[:n])
    ok = sg == 0
    assert np.isfinite(Fz[ok]).all() and np.isfinite(Fu[ok]).all()
    assert np.array_equal(Zp, Zg[perm]) and np.array_equal(Fzp, Fz[perm]) and np.array_equal(Fup, Fu[perm])


@pytest.mark.parametrize("name", ["ant", "quadruped"])
def test_q2_literal_gradients(name):
    """DOJO_FLAG_Q2_LITERAL_GRADIENTS: what get_maximal_gradients!(mechanism, z, u) literally returns (gradients/state.jl:69-76: data
    Jacobian after update_state!, KKT matrix from before it) against the oracle's literal restatement; same forward step as without."""
    from dojo_jl_b200.solver import BatchedStepper, DOJO_FLAG_Q2_LITERAL_GRADIENTS
    from oracle.oracle import Oracle
    mech = dj.get_mechanism(name)
    rng = np.random.default_rng(43)
    B = 24
    Z = jittered_states(mech, B, rng)
    stepper, oracle = BatchedStepper(mech, B), Oracle(mech)
    for _ in range(5):
        Z, _, _ = stepper.step(Z, random_inputs(mech, B, rng))
    U = random_inputs(mech, B, rng)
    Zn, Fz, Fu, sg, ig = stepper.step_grad(Z, U, flags=DOJO_FLAG_Q2_LITERAL_GRADIENTS)
    Zc, Fzc, Fuc, _, _ = stepper.step_grad(Z, U)
    assert np.array_equal(Zn, Zc)
    errs, diff = [], []
    for e in range(B):
        _, Fzo, Fuo, so, io = oracle.step_grad(Z[e], U[e], flags=DOJO_FLAG_Q2_LITERAL_GRADIENTS)
        if so != 0 or sg[e] != 0 or io != ig[e]:
            continue
        sz, su = max(1.0, np.abs(Fzo).max()), max(1.0, np.abs(Fuo).max())
        errs.append(max(np.abs(Fz[e] - Fzo).max() / sz, np.abs(Fu[e] - Fuo).max() / su))
        diff.append(np.abs(Fz[e] - Fzc[e]).max() / sz)
    errs = np.array(errs)
    assert len(errs) >= B // 2
    assert np.median(errs) < 1e-7 and errs.max() < 1e-2, errs
    assert np.median(diff) > 1e-4  # the literal result is a different matrix


@pytest.mark.parametrize("name,B,sample", [("ant", 4096, 768), ("quadruped", 8192, 512)])
def test_parity_on_the_benchmarked_states(name, B, sample):
    """The batch bench.py TIMES (BASELINE C1: ant B = 4096 after its 20-step roll-in in hard contact; C2: quadruped B = 8192, stance
    episodes), not jittered test states: a random subset against the oracle -- identical status, iteration count and contact-mode
    bitmap (gamma_1 > s_1 per contact) for every sampled environment, states to the same-path tolerance.  (Round 1 allowed 3 % of
    the environments a different iteration count; with the joint-limit duals in the joint node the bar is every sampled
    environment.)  bench.py reports the same comparison as rates in its JSON line."""
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    sys.path.insert(0, os.path.join(root, "tools"))
    import bench
    from parity_bench_states import compare
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism(name)
    w = bench.WORKLOADS[name]
    Z, rng = bench.synthetic_batch(mech, B, 0xD0D0 + 1, name)
    steps = w["rollin"] + 3 if not w["episode"] else 5
    U = bench.random_inputs(mech, rng, steps + 1, B, bench.SCALE[name])
    st = BatchedStepper(mech, B)
    for t in range(steps):
        Z, _, _ = st.step(Z, U[t])
    r = compare(mech, Z, U[steps], st, sample, seed=1)
    _record_stats("bench_states_" + name, r)
    assert r["status_mismatch"] == 0 and r["contact_mode_mismatch_all_converged"] == 0, r
    assert r["iters_mismatch"] <= max(1, sample // 200), r          # <= 0.5 %
    assert r["max_abs_dz_same_iters"] <= TOL_SAME_PATH and r["median_abs_dz_same_iters"] <= 1e-11, r


def test_results_do_not_depend_on_the_work_queue_order(monkeypatch):
    """The order in which the environments are dequeued (least likely to stall last, DOJO_B200_LPT) and the line-search assist of the
    drained slots (DOJO_B200_NO_LS_ASSIST) only change WHEN an environment is computed: states, status, iteration counts and solution
    vectors are bit-identical under every setting (B large enough for the order to be used and for the launch to have a tail)."""
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism("ant")
    rng = np.random.default_rng(41)
    B = 1500
    Z = jittered_states(mech, B, rng)
    ref = None
    for env in ({}, {"DOJO_B200_LPT": "0"}, {"DOJO_B200_LPT": "2"}, {"DOJO_B200_NO_LS_ASSIST": "1"}):
        for k in ("DOJO_B200_LPT", "DOJO_B200_NO_LS_ASSIST"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        stepper = BatchedStepper(mech, B)
        Zs, outs = Z, []
        r2 = np.random.default_rng(43)
        for _ in range(6):  # a few steps into contact, where stalls and line-search retries happen
            Zs, st, it, sol = stepper.step(Zs, random_inputs(mech, B, r2, 1.0), return_sol=True)
            outs += [Zs, st, it, sol]
        stepper.close()
        if ref is None:
            ref = outs
        else:
            assert all(np.array_equal(a, b) for a, b in zip(ref, outs)), env
