"""The traced step (dojo_step_trace) on the H100 (run with -m gpu): bit-identical outputs to the untraced step under every work-queue
order, device traces against the oracle's loop heads, the per-class statistics of iteration mismatches on the benchmarked ant batch,
and the verbose printout of api.step / api.simulate."""
import os
import sys

import numpy as np
import pytest

import dojo_jl_b200 as dj
from conftest import jittered_states, random_inputs
from test_gpu_parity import MAX_PATH_FLIPS

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# device against oracle on the same path (equal iteration counts): |device - oracle| <= RTOL |oracle| + ATOL per column (rvio, bvio, alpha,
# mu); nvcc contracts to FMA where the oracle's GCC build contracts elsewhere, so the rows agree to rounding, amplified where a violation
# is the cancellation of O(1) residual entries at the rounding floor
RTOL = 1e-5
ATOL = np.array([1e-11, 1e-11, 0.0, 0.0])


def _rows(tr):
    return int(np.count_nonzero(~np.isnan(tr[:, 4])))


def _close(a, b):
    """rows a, b [n, 5]: trials identical and reals within the tolerance"""
    if not np.array_equal(a[:, 4], b[:, 4]):
        return False
    same = (a[:, :4] == b[:, :4]) | (np.isnan(a[:, :4]) & np.isnan(b[:, :4]))
    return bool((same | (np.abs(a[:, :4] - b[:, :4]) <= RTOL * np.abs(b[:, :4]) + ATOL)).all())


def _into_contact(mech, B, seed, steps=5):
    rng = np.random.default_rng(seed)
    if mech.Nb > 2:
        Z = jittered_states(mech, B, rng)
        U = [random_inputs(mech, B, rng) for _ in range(steps + 1)]
    else:  # a block thrown at the ground
        Z = np.tile(mech.z0, (B, 1))
        Z[:, 2] += rng.uniform(-0.9, 0.0, B)
        Z[:, 3:6] = rng.normal(size=(B, 3)) * [1.0, 1.0, 0.3]
        Z[:, 10:13] = rng.normal(size=(B, 3))
        U = [0.1 * rng.normal(size=(B, mech.nu)) for _ in range(steps + 1)]
    return Z, U


@pytest.mark.parametrize("name,ct,B", [("ant", None, 300), ("quadruped", None, 200), ("atlas", None, 60), ("block", "linear", 200)])
def test_traced_step_is_bit_identical_under_every_order(name, ct, B, monkeypatch):
    """dojo_step_trace == dojo_step bit for bit (states, status, iterations, solutions) a few steps into contact, under the work-queue
    orders (DOJO_B200_LPT), without line-search assist and with the plan tables in global memory; the traces themselves are identical
    under all of these too (block with LinearContact: the DJ_ANY_CONTACT compilation)"""
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism(name, contact_type=ct) if ct else dj.get_mechanism(name)
    Z0, U = _into_contact(mech, B, 7)
    ref = None
    for env in ({}, {"DOJO_B200_LPT": "0"}, {"DOJO_B200_LPT": "2"}, {"DOJO_B200_LPT": "3"}, {"DOJO_B200_NO_LS_ASSIST": "1"},
                {"DOJO_B200_GENERIC_PLAN": "1"}):
        for k in ("DOJO_B200_LPT", "DOJO_B200_NO_LS_ASSIST", "DOJO_B200_GENERIC_PLAN"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        st = BatchedStepper(mech, B)
        Z, outs = Z0, []
        for t in range(len(U)):
            a = st.step(Z, U[t], return_sol=True)
            b = st.step(Z, U[t], return_sol=True, trace=True)
            for x, y in zip(a, b[:4]):
                assert np.array_equal(x, y), (env, t)
            tr = b[4]
            for e in range(B):
                n = _rows(tr[e])
                assert n == (a[2][e] + 1 if a[1][e] == 0 else 50 if a[1][e] == 1 else n), (env, t, e)
                assert np.isnan(tr[e, n:]).all()
            outs += list(b)
            Z = a[0]
        st.close()
        if ref is None:
            ref = outs
        else:
            assert all(np.array_equal(x, y, equal_nan=True) for x, y in zip(ref, outs)), env


def _against_oracle(mech, Z, U, tr, st, it, idx, opts=None):
    """per-class comparison of the device rows with the oracle's for environments idx"""
    from hostemu.trace import TracedOracle
    o = TracedOracle(mech, opts)
    r = {"n": 0, "same_iters": 0, "same_iters_trace_mismatch": 0, "trials_mismatch_same_iters": 0, "iters_mismatch": 0,
         "convergence_test_flips": 0, "line_search_flips": 0, "status_mismatch": 0, "max_rel": 0.0}
    for e in idx:
        so = o.step(Z[e], U[e])[1]
        ot, dt = o.trace(), tr[e, : _rows(tr[e])]
        r["n"] += 1
        if so != st[e]:
            r["status_mismatch"] += 1
            continue
        if dt.shape[0] == ot.shape[0]:
            r["same_iters"] += 1
            if not np.array_equal(dt[:, 4], ot[:, 4]):
                r["trials_mismatch_same_iters"] += 1
            elif not _close(dt, ot):
                r["same_iters_trace_mismatch"] += 1
            big = np.abs(ot[:, :4]) > 1e-10
            d = np.abs(dt[:, :4] - ot[:, :4])
            with np.errstate(invalid="ignore", divide="ignore"):
                rel = np.where(big & ~np.isnan(d), d / np.abs(ot[:, :4]), 0.0)
            r["max_rel"] = max(r["max_rel"], float(rel.max()))
        else:
            r["iters_mismatch"] += 1
            m = min(dt.shape[0], ot.shape[0])
            # a convergence-test flip: the same path up to the shorter trace's last head, where one side's test passed and the other's not
            if _close(dt[:m], ot[:m]):
                r["convergence_test_flips"] += 1
            else:
                r["line_search_flips"] += 1
    return r


def test_device_traces_follow_the_oracle():
    """ant B = 300 into contact: every environment with the oracle's iteration count has the oracle's rows (trials identical, reals
    within RTOL / ATOL); different trial counts at equal iteration counts stay within the path-flip budget of the parity tests"""
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism("ant")
    B = 300
    Z, U = _into_contact(mech, B, 11)
    st = BatchedStepper(mech, B)
    for t in range(len(U) - 1):
        Z = st.step(Z, U[t])[0]
    Zn, s, it, tr = st.step(Z, U[-1], trace=True)
    r = _against_oracle(mech, Z, U[-1], tr, s, it, range(B))
    print("trace_vs_oracle ant B=300", r)
    assert r["status_mismatch"] == 0, r
    assert r["trials_mismatch_same_iters"] <= max(1, MAX_PATH_FLIPS * B), r
    assert r["same_iters_trace_mismatch"] == 0, r
    assert r["line_search_flips"] + r["trials_mismatch_same_iters"] <= max(1, MAX_PATH_FLIPS * B), r


def test_statistics_on_the_benchmarked_ant_states():
    """bench.py's ant batch (B = 4096 after its roll-in): per-class statistics of the iteration mismatches against the oracle on a
    sample, and the line-search trials of the environments that end :failed (the stalls that set the length of a per-step launch)"""
    sys.path.insert(0, ROOT)
    import bench
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism("ant")
    w = bench.WORKLOADS["ant"]
    B = 4096
    Z, rng = bench.synthetic_batch(mech, B, 0xD0D0 + 1, "ant")
    steps = w["rollin"] + 3
    U = bench.random_inputs(mech, rng, steps + 1, B, bench.SCALE["ant"])
    st = BatchedStepper(mech, B)
    for t in range(steps):
        Z = st.step(Z, U[t])[0]
    Zn, s, it, tr = st.step(Z, U[steps], trace=True)
    sample = np.sort(np.random.default_rng(1).choice(B, size=512, replace=False))
    r = _against_oracle(mech, Z, U[steps], tr, s, it, sample)
    failed = np.flatnonzero(s == 1)
    trials = tr[failed, 1:, 4].ravel()
    trials = trials[~np.isnan(trials)].astype(int)
    hist = np.bincount(trials, minlength=11)[1:].tolist() if trials.size else []
    stalled = int(sum((tr[e, 1:_rows(tr[e]), 4] == 10).mean() > 0.5 for e in failed))
    print("bench_states_ant_trace", {"B": B, **r, "failed": int(failed.size), "failed_stalled": stalled,
                                     "failed_trials_hist_1_to_10": hist, "mean_iters": float(it.mean()), "max_iters": int(it.max())})
    assert r["status_mismatch"] == 0 and r["same_iters_trace_mismatch"] == 0, r


def test_api_step_verbose_prints_the_table(capsys):
    """api.step with SolverOptions(verbose=True) and one environment prints header + one line per loop head; a batch prints nothing;
    api.simulate prints one table per step and returns what the fused rollout returns"""
    from dojo_jl_b200 import api
    mech = dj.get_mechanism("ant")
    g = np.load(os.path.join(ROOT, "tests", "golden", "ant.npz"))
    quiet, loud = api.SolverOptions(), api.SolverOptions(verbose=True)
    zq = api.step(mech, g["Z"][0], g["U"][0], opts=quiet)
    assert capsys.readouterr().out == ""
    zl = api.step(mech, g["Z"][0], g["U"][0], opts=loud)
    out = capsys.readouterr().out.split("\n")
    assert np.array_equal(zq, zl)
    _, _, iters = api.step(mech, g["Z"][:1], g["U"][:1], opts=quiet)
    assert out[1] == "n    bvio    rvio     α       μ" and len([x for x in out[3:] if x]) == iters[0] + 1
    assert out[3].startswith("1   ") and out[3].endswith(" 1e+0    0e+0")
    api.step(mech, g["Z"][:2], g["U"][:2], opts=loud)
    assert capsys.readouterr().out == ""
    zf = api.simulate(mech, 3, z0=g["Z"][0], opts=quiet)
    zv = api.simulate(mech, 3, z0=g["Z"][0], opts=loud)
    printed = capsys.readouterr().out
    assert np.array_equal(zf, zv) and printed.count("n    bvio    rvio") == 3
    print(printed)


def test_host_and_device_pointer_traces_agree():
    """dojo_step_trace with host buffers (staged) == dojo_step_trace_async with device buffers; a budget of 0 iterations gives an empty
    trace, and a missing trace buffer is refused"""
    import ctypes as C
    import torch
    from dojo_jl_b200 import capi
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism("quadruped")
    g = np.load(os.path.join(ROOT, "tests", "golden", "quadruped.npz"))
    Z, U = g["Z"], g["U"]
    B = Z.shape[0]
    st = BatchedStepper(mech, 16)
    Zn, s, it, tr = st.step(Z, U, trace=True)
    dev = torch.device("cuda:0")
    dZ, dU = torch.from_numpy(Z).to(dev), torch.from_numpy(U).to(dev)
    dZn, dst, dit = torch.empty_like(dZ), torch.empty(B, dtype=torch.int32, device=dev), torch.empty(B, dtype=torch.int32, device=dev)
    dtr = torch.empty((B, 50, 5), dtype=torch.float64, device=dev)
    st.step_device(dZ.data_ptr(), dU.data_ptr(), dZn.data_ptr(), B, dstatus=dst.data_ptr(), diters=dit.data_ptr(), dtrace=dtr.data_ptr(),
                   stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(dZn.cpu().numpy(), Zn) and np.array_equal(dit.cpu().numpy(), it)
    assert np.array_equal(dtr.cpu().numpy(), tr, equal_nan=True)
    Z0, s0, it0, tr0 = st.step(Z, U, opts=capi.solver_options(max_iter=0), trace=True)
    assert tr0.shape == (B, 0, 5) and (s0 == 1).all() and (it0 == 0).all()
    o = capi.solver_options()
    rc = st.L.dojo_step_trace(st.h, C.byref(o), B, C.c_void_p(Z.ctypes.data), C.c_void_p(U.ctypes.data), None,
                              C.c_void_p(Zn.ctypes.data), None, None, None, None, 0)
    assert rc == -1
