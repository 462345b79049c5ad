"""The traced step (dojo_step_trace): the solver's per-iteration record, on the kernel emulation against the oracle.

The traced kernel (dojo_step_kernel<false, PLAN_SMEM, true>) runs the same Newton loop as the untraced one and also writes one row per
loop-head test, [rvio, bvio, alpha, mu, trials], where alpha, mu and trials belong to the iteration before the head (the columns
mehrotra! prints with verbose = true, plus the line-search trial count).  Checked here on the CPU with the product's kernel source
(tests/hostemu):
  * its outputs are bit-identical to the untraced kernel's;
  * its rows are the oracle's loop heads: the same row count, identical trials, reals within TRACE_RTOL;
  * the row-count rules, the NaN padding and row 0;
  * the oracle build that records the trials (tests/hostemu/trace.py) is the oracle;
  * the trace does not depend on the thread order nor on the line-search assist;
  * the table api.format_solver_trace prints, on oracle traces."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import dojo_jl_b200 as dj
from dojo_jl_b200 import capi
from dojo_jl_b200.api import _scn, format_solver_trace
from oracle.oracle import Oracle

from conftest import jittered_states, random_inputs
from hostemu.trace import TracedEmu, TracedOracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
# Tolerance of the emulated trace against the oracle's: |device - oracle| <= TRACE_RTOL |oracle| + TRACE_ATOL, column by column (rvio,
# bvio, alpha, mu).  The two compute the same quantities in different orders (the oracle is another restatement of mehrotra!, compiled
# with FMA contraction; the emulation has none), so they agree to rounding.  Measured over the cases below: alpha and mu within 6.2e-9
# relative, violations above 1e-6 within 2.7e-10 relative, and violations below 1e-10 -- the converged heads, at the rounding floor of
# O(1) residual entries -- within 5.3e-15 absolute.
TRACE_RTOL = 1e-7
TRACE_ATOL = np.array([1e-13, 1e-13, 0.0, 0.0])


def _thrown(mech, B, rng):
    Z = np.tile(mech.z0, (B, 1))
    Z[:, 2] += rng.uniform(-0.4 if mech.name == "sphere" else -0.9, 0.0, B)
    Z[:, 3:6] = rng.normal(size=(B, 3)) * [1.0, 1.0, 0.3]
    Z[:, 10:13] = rng.normal(size=(B, 3))
    return Z, 0.1 * rng.normal(size=(B, mech.nu))


def _case(name, ct):
    """(mechanism, Z, U): the golden fixtures, or a few steps into contact for the small models"""
    if ct is None and os.path.exists(os.path.join(GOLDEN, name + ".npz")):
        g = np.load(os.path.join(GOLDEN, name + ".npz"))
        return dj.get_mechanism(name), g["Z"], g["U"]
    mech = dj.get_mechanism(name, contact_type=ct) if ct else dj.get_mechanism(name)
    rng = np.random.default_rng(5)
    o = Oracle(mech)
    if name == "raiberthopper":
        Z, U = np.tile(mech.z0, (3, 1)), random_inputs(mech, 3, rng, 0.3)
    else:
        Z, U = _thrown(mech, 3, rng)
    for _ in range(8):  # into contact
        Z = np.stack([o.step(Z[e], U[e])[0] for e in range(Z.shape[0])])
    return mech, Z, U


def _rows(tr):
    return int(np.count_nonzero(~np.isnan(tr[:, 4])))


def _check_rows(tr, st, it, max_iter):
    """the row-count rules and the NaN padding of one environment's trace"""
    n = _rows(tr)
    if st == 0:
        assert n == it + 1
    elif st == 1:
        assert n == it == max(max_iter, 0)
    # mu may be NaN at a head: without cones the centering ratio is 0 / 0, and max(NaN, x) = NaN in Julia (solver/mehrotra.jl:44-47)
    assert np.isnan(tr[n:]).all() and not np.isnan(tr[:n, [2, 4]]).any()
    if n:
        assert tuple(tr[0, 2:]) == (1.0, 0.0, 0.0)
        assert (tr[1:n, 4] >= 1).all() and (tr[1:n, 4] == np.round(tr[1:n, 4])).all()
    return n


def _compare_with_oracle(o, z, u, opts, tr, st, it):
    """one environment: the emulated trace against the oracle's loop heads.  Returns the largest relative difference of the entries
    above 1e-10 and the largest absolute difference of the others."""
    zo, so, io = o.step(z, u, opts=opts)
    ot = o.trace()
    assert (st, it) == (so, io)
    n = _check_rows(tr, st, it, opts.max_iter)
    assert ot.shape == (n, 5)
    assert np.array_equal(tr[:n, 4], ot[:, 4])
    d = np.abs(tr[:n, :4] - ot[:, :4])
    d[(tr[:n, :4] == ot[:, :4]) | (np.isnan(tr[:n, :4]) & np.isnan(ot[:, :4]))] = 0.0
    same = (tr[:n, :4] == ot[:, :4]) | (np.isnan(tr[:n, :4]) & np.isnan(ot[:, :4]))
    assert (same | (d <= TRACE_RTOL * np.abs(ot[:, :4]) + TRACE_ATOL)).all(), d
    if not n:
        return 0.0, 0.0
    big = np.abs(ot[:, :4]) > 1e-10
    rel = np.where(big, d / np.where(big, np.abs(ot[:, :4]), 1.0), 0.0)
    return float(rel.max()), float(np.where(big, 0.0, d).max())


def test_traced_oracle_is_the_oracle():
    """the oracle's build with the trials column (hostemu/trace.py): the same steps bit for bit, the same first four columns of every
    row, and a fifth column of trial counts (0 in row 0, then 1 .. max_ls)"""
    for name, ct in (("ant", None), ("block", "linear")):
        mech, Z, U = _case(name, ct)
        o, t = Oracle(mech), TracedOracle(mech)
        for e in range(Z.shape[0]):
            a, b = o.step(Z[e], U[e], return_sol=True), t.step(Z[e], U[e], return_sol=True)
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
            tr = t.trace()
            assert np.array_equal(o.trace(), tr[:, :4], equal_nan=True) and tr.shape == (a[2] + 1, 5)
            assert tr[0, 4] == 0 and ((tr[1:, 4] >= 1) & (tr[1:, 4] <= 10)).all()


CASES = [("pendulum", None), ("ant", None), ("quadruped", None), ("atlas", None), ("block", "linear"), ("block", "impact"),
         ("sphere", "linear"), ("sphere", "impact"), ("raiberthopper", None)]


@pytest.mark.parametrize("name,ct", CASES)
def test_traced_step_is_the_untraced_step_and_follows_the_oracle(name, ct):
    mech, Z, U = _case(name, ct)
    em, o = TracedEmu(mech), TracedOracle(mech)
    opts = capi.solver_options()
    slots = 2 if mech.Nb > 13 else 4
    Zn, st, it, sol = em.step(Z, U, opts, slots=slots)
    Zt, stt, itt, solt, tr = em.step_trace(Z, U, opts, slots=slots)
    assert np.array_equal(Zn, Zt) and np.array_equal(st, stt) and np.array_equal(it, itt) and np.array_equal(sol, solt)
    assert tr.shape == (Z.shape[0], opts.max_iter, 5)
    d = np.array([_compare_with_oracle(o, Z[e], U[e], opts, tr[e], st[e], it[e]) for e in range(Z.shape[0])])
    print(f"{name} {ct or ''}: iterations {it.tolist()}, trace against the oracle: relative difference {d[:, 0].max():.1e}, "
          f"absolute difference of entries below 1e-10 {d[:, 1].max():.1e}")


def test_failed_solves_record_max_iter_rows_and_stalled_trials(monkeypatch):
    """unreachable tolerances: the solve ends :failed with max_iter rows; the trace is the same with and without line-search assist
    (trials come from the owner's count)"""
    mech = dj.get_mechanism("ant")
    rng = np.random.default_rng(3)
    Z = jittered_states(mech, 1, rng)
    oo = Oracle(mech)
    for _ in range(8):
        Z = np.stack([oo.step(Z[0], random_inputs(mech, 1, rng)[0])[0]])
    U = random_inputs(mech, 1, rng)
    opts = capi.solver_options(rtol=1e-14, btol=1e-14, max_iter=12)
    monkeypatch.delenv("DOJO_B200_NO_LS_ASSIST", raising=False)
    on = TracedEmu(mech)
    monkeypatch.setenv("DOJO_B200_NO_LS_ASSIST", "1")
    off = TracedEmu(mech)
    monkeypatch.delenv("DOJO_B200_NO_LS_ASSIST", raising=False)
    a, b = on.step_trace(Z, U, opts, slots=4), off.step_trace(Z, U, opts, slots=4)  # B = 1: three helper slots from the first iteration
    for x, y in zip(a, b):
        assert np.array_equal(x, y, equal_nan=True)
    Zn, st, it, sol, tr = a
    assert st[0] == 1 and it[0] == opts.max_iter
    # past the rounding floor the iterates are rounding noise, so only the row rules are held here (the oracle comparison of
    # failed solves with reachable iterates: test_row_zero_short_budgets_and_nonfinite)
    assert _check_rows(tr[0], st[0], it[0], opts.max_iter) == opts.max_iter
    # several environments with tight tolerances: the helpers join at the tail of the launch
    g = np.load(os.path.join(GOLDEN, "ant.npz"))
    opts = capi.solver_options(rtol=1e-9, btol=1e-9)
    a, b = on.step_trace(g["Z"][:3], g["U"][:3], opts, slots=4), off.step_trace(g["Z"][:3], g["U"][:3], opts, slots=4)
    for x, y in zip(a, b):
        assert np.array_equal(x, y, equal_nan=True)


def test_row_zero_short_budgets_and_nonfinite():
    mech = dj.get_mechanism("quadruped")
    g = np.load(os.path.join(GOLDEN, "quadruped.npz"))
    Z, U = g["Z"][:2], g["U"][:2]
    em, o = TracedEmu(mech), TracedOracle(mech)
    # row 0 = (initial rvio, bvio, 1, 0, 0), the oracle's first head
    Zn, st, it, sol, tr = em.step_trace(Z, U, slots=2)
    o.step(Z[0], U[0])
    ot = o.trace()
    assert np.allclose(tr[0, 0, :2], ot[0, :2], rtol=TRACE_RTOL, atol=0) and tuple(tr[0, 0, 2:]) == (1.0, 0.0, 0.0)
    # a budget of 2 iterations: :failed with exactly 2 rows; a budget of 0 or less: no row at all (the loop body never runs)
    for max_iter in (2, 1, 0, -1):
        opts = capi.solver_options(max_iter=max_iter)
        Zn, st, it, sol, tr = em.step_trace(Z, U, opts, slots=2)
        assert tr.shape == (2, max(max_iter, 0), 5)
        for e in range(2):
            _compare_with_oracle(o, Z[e], U[e], opts, tr[e], st[e], it[e])
    # a non-finite state: the heads actually reached (row 0 only), like the oracle
    Zb = Z.copy()
    Zb[1, 3] = np.nan
    Zn, st, it, sol, tr = em.step_trace(Zb, U, slots=2)
    o.step(Zb[1], U[1])
    assert st[1] == 3 and _rows(tr[1]) == o.trace().shape[0] == 1 and np.isnan(tr[1, 1:]).all()
    assert st[0] == 0 and _rows(tr[0]) == it[0] + 1


ORDER_SCRIPT = r"""
import sys, numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests")
import dojo_jl_b200 as dj
from dojo_jl_b200 import capi
from hostemu.trace import TracedEmu
from conftest import jittered_states, random_inputs
out = {}
for name, kw in (("ant", {}), ("block", {"contact_type": "linear"})):
    m = dj.get_mechanism(name, **kw)
    rng = np.random.default_rng(23)
    Z = jittered_states(m, 3, rng) if m.Nb > 2 else np.tile(m.z0, (3, 1))
    U = random_inputs(m, 3, rng)
    for tight in (False, True):
        opts = capi.solver_options(rtol=1e-9, btol=1e-9) if tight else None
        r = TracedEmu(m).step_trace(Z, U, opts, slots=4)
        for k, v in zip(("Zn", "st", "it", "sol", "trace"), r):
            out["%%s_%%d_%%s" %% (name, tight, k)] = v
np.savez(sys.argv[1], **out)
"""


def _run_order(order, path):
    env = dict(os.environ)
    env.pop("HOSTEMU_ORDER", None)
    if order:
        env["HOSTEMU_ORDER"] = order
    r = subprocess.run([sys.executable, "-c", ORDER_SCRIPT % {"root": ROOT}, path], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    return np.load(path)


def test_trace_does_not_depend_on_the_thread_order(tmp_path):
    ref = _run_order(None, str(tmp_path / "asc.npz"))
    for order in ("reverse", "random"):
        got = _run_order(order, str(tmp_path / (order + ".npz")))
        for k in ref.files:
            assert np.array_equal(ref[k], got[k], equal_nan=True), (order, k)


# ---------------------------------------------------------------------------------------------------------------- the printed table
def test_scn_matches_the_reference_rules():
    """scn(a, digits=0) (utilities/methods.jl:9-43): mantissa rounded to an integer, 10 carried into the exponent,
    a blank in front of non-negative numbers, exponent with its sign and without padding"""
    assert _scn(1.0) == " 1e+0"
    assert _scn(0.0) == " 0e+0"
    assert _scn(3.7e-5) == " 4e-5"
    assert _scn(9.6e-3) == " 1e-2"
    assert _scn(2.4e-7) == " 2e-7"
    assert _scn(-2.6e3) == "-3e+3"
    assert _scn(123.0) == " 1e+2"
    assert _scn(1e-12) == " 1e-12"
    assert _scn(float("nan")) == " NaN "
    assert _scn(float("inf")) == " Inf" and _scn(-float("inf")) == "-Inf"


def test_formatted_table_of_oracle_traces():
    """header and one line per loop head, `n   bvio   rvio   α   μ` (bvio before rvio, as solver_status prints them)"""
    mech = dj.get_mechanism("ant")
    g = np.load(os.path.join(GOLDEN, "ant.npz"))
    o = TracedOracle(mech)
    for opts in (capi.solver_options(), capi.solver_options(rtol=1e-14, btol=1e-14, max_iter=5)):
        o.step(g["Z"][0], g["U"][0], opts=opts)
        ot = o.trace()
        tr = np.full((opts.max_iter, 5), np.nan)
        tr[: ot.shape[0]] = ot
        lines = format_solver_trace(tr).split("\n")
        assert lines[0] == " " * 49 and lines[1] == "n    bvio    rvio     α       μ" and lines[2] == "–" * 49
        assert len(lines) == 3 + ot.shape[0]
        num = r"( \d|-\d)e[+-]\d+"
        for r, line in enumerate(lines[3:]):
            assert re.fullmatch(r"\d+" + ("   " + num) * 4, line), line
            assert line == f"{r + 1}   {_scn(ot[r, 1])}   {_scn(ot[r, 0])}   {_scn(ot[r, 2])}   {_scn(ot[r, 3])}"
        assert lines[3].endswith(" 1e+0    0e+0")  # row 0: alpha = 1, mu = 0
    assert format_solver_trace(np.full((4, 5), np.nan)).count("\n") == 2  # no head reached: the header only
