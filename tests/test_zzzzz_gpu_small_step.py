"""The forward kernel specialised for small mechanisms on the H100 (run with -m gpu): dojo_create selects it for ant, quadruped and
pendulum and nowhere else, and it is bit-identical to the generic kernel (DOJO_B200_GENERIC_STEP) on the states bench.py times --
states, status, Newton iterations and solution vectors of steps and fused rollouts, and the gradients of dojo_step_grad, whose forward
launch runs it.  The CPU twin is tests/test_small_step.py."""
import os
import sys

import numpy as np
import pytest

import dojo_jl_b200 as dj

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _stepper(mech, B, generic, monkeypatch):
    from dojo_jl_b200.solver import BatchedStepper
    if generic:
        monkeypatch.setenv("DOJO_B200_GENERIC_STEP", "1")
    else:
        monkeypatch.delenv("DOJO_B200_GENERIC_STEP", raising=False)
    st = BatchedStepper(mech, B)
    monkeypatch.delenv("DOJO_B200_GENERIC_STEP", raising=False)
    return st


def _bench_states(name, B):
    """bench.py's timed state of the workload: its seeded batch after its roll-in, and the inputs of the first timed steps"""
    import torch
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import bench
    from dojo_jl_b200 import capi
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism(name)
    w = bench.WORKLOADS[name]
    Z0, rng = bench.synthetic_batch(mech, B, 0xD0D0 + 1, name)
    U = torch.from_numpy(bench.random_inputs(mech, rng, w["rollin"] + 4, B, bench.SCALE.get(name, 1.0))).cuda()
    Za = torch.from_numpy(Z0).cuda()
    Zb = torch.empty_like(Za)
    st = BatchedStepper(mech, B)
    for t in range(w["rollin"]):
        st.step_device(Za.data_ptr(), U[t].data_ptr(), Zb.data_ptr(), B, capi.solver_options())
        Za, Zb = Zb, Za
    torch.cuda.synchronize()
    return mech, Za, U[w["rollin"]:]


@pytest.mark.parametrize("name,small", [("ant", 1), ("quadruped", 1), ("pendulum", 1), ("atlas", 0)])
def test_selection(name, small, monkeypatch):
    for k in ("DOJO_B200_WARPS", "DOJO_B200_NO_JOINT_PAIR", "DOJO_B200_NO_LS_PAIR", "DOJO_B200_GLOBAL_PLAN", "DOJO_B200_GENERIC_PLAN"):
        monkeypatch.delenv(k, raising=False)
    m = dj.get_mechanism(name)
    assert _stepper(m, 8, False, monkeypatch).launch_config["small_step"] == small
    assert _stepper(m, 8, True, monkeypatch).launch_config["small_step"] == 0
    if small:
        for env in ({"DOJO_B200_GENERIC_PLAN": "1"}, {"DOJO_B200_GLOBAL_PLAN": "1"}, {"DOJO_B200_NO_JOINT_PAIR": "1"}, {"DOJO_B200_WARPS": "4"}):
            for k, v in env.items():
                monkeypatch.setenv(k, v)
            assert _stepper(m, 8, False, monkeypatch).launch_config["small_step"] == 0, env
            for k in env:
                monkeypatch.delenv(k)


@pytest.mark.parametrize("name,B", [("ant", 4096), ("quadruped", 8192)])
def test_bench_states_are_bit_identical(name, B, monkeypatch):
    """three steps from bench.py's timed state with both kernels: states, status, iterations and solution vectors bit for bit"""
    import torch
    mech, Z, U = _bench_states(name, B)
    arms = {g: _stepper(mech, B, g, monkeypatch) for g in (True, False)}
    assert arms[False].launch_config["small_step"] == 1 and arms[True].launch_config["small_step"] == 0
    for t in range(3):
        out = {}
        for g, st in arms.items():
            zn = torch.empty_like(Z)
            s, it = torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda")
            sol = torch.empty((B, mech.nres), dtype=torch.float64, device="cuda")
            st.step_device(Z.data_ptr(), U[t].data_ptr(), zn.data_ptr(), B, dstatus=s.data_ptr(), diters=it.data_ptr(), dsol=sol.data_ptr())
            out[g] = (zn, s, it, sol)
        torch.cuda.synchronize()
        for k, what in enumerate(("states", "status", "iterations", "solutions")):
            a, b = out[True][k], out[False][k]
            assert torch.equal(a, b), f"{name} step {t}: {what} differ ({int((a != b).sum())} entries)"
        print(f"{name} B={B} step {t}: mean iterations {out[False][2].float().mean().item():.3f}, failed {int((out[False][1] != 0).sum())}")
        Z = out[True][0]


def test_rollouts_are_bit_identical(monkeypatch):
    import torch
    B, T = 1024, 4
    mech, Z, U = _bench_states("ant", B)
    U = U[:T].contiguous()
    res = {}
    for g in (True, False):
        st = _stepper(mech, B, g, monkeypatch)
        zf = torch.empty_like(Z)
        traj = torch.empty((T, B, mech.nz), dtype=torch.float64, device="cuda")
        s = torch.zeros(B, dtype=torch.int32, device="cuda")
        st.rollout_device(Z.data_ptr(), U.data_ptr(), zf.data_ptr(), B, T, dtraj=traj.data_ptr(), dstatus=s.data_ptr())
        torch.cuda.synchronize()
        res[g] = (zf, traj, s)
    for a, b in zip(res[True], res[False]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("name,B", [("ant", 1024), ("quadruped", 512)])
def test_gradients_are_bit_identical(name, B, monkeypatch):
    """dojo_step_grad: the forward launch runs the specialised kernel, the gradient kernel reads its solutions"""
    import torch
    mech, Z, U = _bench_states(name, B)
    ng = 12 * mech.Nb
    res = {}
    for g in (True, False):
        st = _stepper(mech, B, g, monkeypatch)
        zn = torch.empty_like(Z)
        Fz = torch.empty((B, ng, ng), dtype=torch.float64, device="cuda")
        Fu = torch.empty((B, mech.nu, ng), dtype=torch.float64, device="cuda")
        s, it = torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda")
        st.step_grad_device(Z.data_ptr(), U[0].data_ptr(), zn.data_ptr(), Fz.data_ptr(), Fu.data_ptr(), B, dstatus=s.data_ptr(), diters=it.data_ptr())
        torch.cuda.synchronize()
        res[g] = (zn, Fz, Fu, s, it)
    for k, what in enumerate(("states", "Fz", "Fu", "status", "iterations")):
        a, b = res[True][k], res[False][k]
        assert torch.equal(a, b) or (what in ("Fz", "Fu") and torch.equal(torch.nan_to_num(a, nan=7.0), torch.nan_to_num(b, nan=7.0))), \
            f"{name}: {what} differ"
