"""The boundary shapes of tests/test_shape_boundaries.py on the H100 (run with -m gpu), through the C-ABI (BatchedStepper):
parity with the oracle, the launch configuration each shape is meant to reach, batch sizes around the slot and SM counts,
the diagnostic switches (bit-identical results), the chunked host-pointer gradient staging, and the refusals."""
import numpy as np
import pytest

import dojo_jl_b200 as dj
from conftest import jittered_states, random_inputs
from test_gpu_parity import _compare_rollout
from test_shape_boundaries import EXPECTED, SWITCHES, shape

pytestmark = pytest.mark.gpu

DOJO_EINVAL, DOJO_ENOMEM = -1, -3
NO_GRAD = ("big_nograd", "cm32")  # gradient workspace larger than the shared memory of one SM
# where the plan tables live on the H100 (forward, gradient): all of them behind the arenas ("full"), a prefix ("partial") or
# none (global memory).  The gradient launches of w16 / c17 / star32 copy a prefix, chain32's workspace leaves no room at all.
PLAN = {"one_body_32c": ("full", "full"), "w16": ("full", "partial"), "b17": ("full", "full"), "c17": ("full", "partial"),
        "chain32": ("full", "none"), "star32": ("full", "partial"), "big_nograd": ("full", None), "cm32": ("full", None)}


def _placement(mask):
    return "full" if mask == 0xff else "none" if mask == 0 else "partial"


def _states(m, B, seed):
    rng = np.random.default_rng(seed)
    Z = jittered_states(m, B, rng, base_z=(0.0, 0.05)) if m.Nb > 1 else np.tile(m.z0, (B, 1))
    return Z, rng


@pytest.mark.parametrize("name", list(EXPECTED))
def test_launch_configuration(name):
    """what dojo_create picks on the H100 for each shape (warps, paired line search, slots, plan placement, gradient chunk)"""
    import torch
    from dojo_jl_b200.solver import BatchedStepper
    m = shape(name)
    st = BatchedStepper(m, 8)
    cfg = st.launch_config
    print("launch_config", name, cfg)
    _, _, nw, ls_pair, _, chunk = EXPECTED[name]
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    assert cfg["warps_per_env"] == nw and cfg["ls_pair"] == ls_pair
    assert cfg["slots"] == max(1, min(optin // cfg["arena_bytes"], 256 // (32 * nw), 8))
    fwd, grad = PLAN[name]
    assert _placement(cfg["plan_smem_mask"]) == fwd, f"{name}: the forward plan is no longer placed '{fwd}' in shared memory"
    if name in NO_GRAD:
        assert cfg["grad_arena_bytes"] == 0
    else:
        assert cfg["grad_chunk"] == chunk and 0 < cfg["grad_arena_bytes"] <= optin
        assert _placement(cfg["plan_smem_mask_grad"]) == grad, f"{name}: the gradient plan is no longer placed '{grad}' in shared memory"
    if name == "chain32":
        assert cfg["phases"] >= 60
    st.close()


@pytest.mark.parametrize("name", list(EXPECTED))
def test_step_parity_with_oracle(name):
    """a short rollout under random inputs against the oracle, at the bar of tests/test_gpu_parity.py::test_step_parity"""
    m = shape(name)
    _compare_rollout(m, 24, 4, seed=7, scale=0.5, tol_median=1e-11)


def _gradient_parity(m, st, B, seed):
    """dojo_step_grad after a few steps against the oracle, at the bar of tests/test_gpu_parity.py::test_gradient_parity.
    Returns the last states and the input generator."""
    from oracle.oracle import Oracle
    Z, rng = _states(m, B, seed)
    o = Oracle(m)
    for _ in range(3):
        Z, _, _ = st.step(Z, random_inputs(m, B, rng, 0.5))
    U = random_inputs(m, B, rng, 0.5)
    Zn, Fz, Fu, sg, ig = st.step_grad(Z, U)
    assert np.array_equal(Zn, st.step(Z, U)[0])
    errs = []
    for e in range(B):
        _, Fzo, Fuo, so, io = o.step_grad(Z[e], U[e])
        if so != 0 or sg[e] != 0 or io != ig[e]:
            continue
        errs.append(max(np.abs(Fz[e] - Fzo).max() / max(1.0, np.abs(Fzo).max()), np.abs(Fu[e] - Fuo).max() / max(1.0, np.abs(Fuo).max())))
    errs = np.array(errs)
    print("gradient_parity", m.name, errs)
    assert len(errs) >= B // 2
    assert np.median(errs) < 1e-7 and np.quantile(errs, 0.9) < 1e-4 and errs.max() < 1e-2, errs
    return Z, rng


@pytest.mark.parametrize("name", [n for n in EXPECTED if n not in NO_GRAD])
def test_gradient_parity_with_oracle(name):
    """at the bar of tests/test_gpu_parity.py::test_gradient_parity; fused rollout equals the steps bit for bit"""
    from dojo_jl_b200.solver import BatchedStepper
    m = shape(name)
    B = 8
    st = BatchedStepper(m, B)
    Z, rng = _gradient_parity(m, st, B, 21)
    T = 4
    UT = np.stack([random_inputs(m, B, rng, 0.5) for _ in range(T)])
    Zf, _, traj = st.rollout(Z, UT, T, record=True)
    Zs = Z
    for t in range(T):
        Zs = st.step(Zs, UT[t])[0]
        assert np.array_equal(traj[t], Zs)
    assert np.array_equal(Zf, Zs)


@pytest.mark.parametrize("name", ["w16", "b17", "chain32"])
def test_batch_boundaries(name):
    """B in {1, slots - 1, slots, slots + 1, SMs x slots, SMs x slots + 1}: every row bit-identical to the same environment in
    one larger batch"""
    import torch
    from dojo_jl_b200.solver import BatchedStepper
    m = shape(name)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    probe = BatchedStepper(m, 1)
    slots = probe.launch_config["slots"]
    probe.close()
    sizes = sorted({1, max(1, slots - 1), slots, slots + 1, sm * slots, sm * slots + 1})
    Bmax = sizes[-1] + 3
    Z, rng = _states(m, 16, 33)
    Z = Z[rng.integers(0, 16, Bmax)]
    U = random_inputs(m, Bmax, rng, 0.5)
    st = BatchedStepper(m, Bmax)
    Zf, sf, itf, solf = st.step(Z, U, return_sol=True)
    for b in sizes:
        Zb, sb, itb, solb = st.step(Z[:b], U[:b], return_sol=True)
        assert np.array_equal(Zb, Zf[:b]) and np.array_equal(sb, sf[:b]) and np.array_equal(itb, itf[:b]) and np.array_equal(solb, solf[:b]), b
    st.close()


DEFAULT_WARPS = {"ant": 2, "w16": 2, "b17": 4, "chain32": 4}
GPU_SWITCHES = [{}, {"DOJO_B200_NO_LS_PAIR": "1"}, {"DOJO_B200_GLOBAL_PLAN": "1"}, {"DOJO_B200_GENERIC_PLAN": "1"}, {"DOJO_B200_SLOTS": "1"},
                {"DOJO_B200_NO_GRAD_OVERLAP": "1"}]


def _mech(name):
    return dj.get_mechanism(name) if name == "ant" else shape(name)


def _set_switches(monkeypatch, env):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("name", ["ant", "w16", "b17", "chain32"])
def test_switches_leave_results_bit_identical(name, monkeypatch):
    """forward outputs (states, status, iterations, solution vectors) and gradients under each diagnostic switch, against the
    default: cross-checks the TMA-copied plan, the PLAN_SMEM kernel variant and the programmatic-launch overlap against the
    alternatives.  (Another warp count and the one-lane joint assembly change rounding: next test.)"""
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech(name)
    B = 300
    Z, rng = _states(m, 32, 41)
    Z = Z[rng.integers(0, 32, B)]
    U = [random_inputs(m, B, rng, 0.5) for _ in range(3)]
    ref, differ = None, []
    for env in GPU_SWITCHES + [{"DOJO_B200_WARPS": str(DEFAULT_WARPS[name])}]:
        _set_switches(monkeypatch, env)
        st = BatchedStepper(m, B)
        cfg = st.launch_config
        assert cfg["warps_per_env"] == DEFAULT_WARPS[name]
        if env == {"DOJO_B200_GLOBAL_PLAN": "1"}:
            assert cfg["plan_smem_mask"] == 0
        Zs, outs = Z, []
        for t in range(3):
            Zs, s, it, sol = st.step(Zs, U[t], return_sol=True)
            outs += [Zs, s, it, sol]
        outs += list(st.step_grad(Z, U[0]))
        st.close()
        if ref is None:
            ref = outs
        elif not all(np.array_equal(a, b) for a, b in zip(ref, outs)):
            differ.append(env)
    assert not differ, differ


ROUNDING_SWITCHES = [{"DOJO_B200_NO_JOINT_PAIR": "1"}] + [{"DOJO_B200_WARPS": w} for w in ("1", "2", "4", "8")]


@pytest.mark.parametrize("env", ROUNDING_SWITCHES, ids=lambda env: ",".join(f"{k[10:]}={v}" for k, v in env.items()))
@pytest.mark.parametrize("name", ["ant", "w16", "b17", "chain32"])
def test_switches_that_change_rounding_match_oracle(name, env, monkeypatch):
    """Two switches change results in the last bits, so they are held to the oracle: steps at the bar of
    tests/test_gpu_parity.py::test_step_parity, gradients at the bar of test_gradient_parity.
      * A warp count other than the default: block_sum3 (dojo_kernels.cuh) sums the complementarity products that set the
        centering parameter per lane over the nodes warp_roles gives it, then the per-warp partials in warp order, so the
        order of that sum follows the warp count.  8 warps run the gradient kernel with an 8-column chunk (one column per warp).
      * DOJO_B200_NO_JOINT_PAIR: each joint assembled on one lane by eval_joint instead of two by eval_joint_pair, the same
        set_entries! terms in another instruction stream that nvcc contracts into fused multiply-adds differently (with
        -fmad=false the two are bit-identical, as on the emulation).
    The gradient chunk never gets narrower than the warp count."""
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech(name)
    w = env.get("DOJO_B200_WARPS")
    if w is not None and int(w) == DEFAULT_WARPS[name]:
        pytest.skip("the default warp count is in the bit-identical matrix")
    _set_switches(monkeypatch, env)
    B = 8
    st = BatchedStepper(m, B)
    cfg = st.launch_config
    if w is not None:
        assert cfg["warps_per_env"] == int(w) and cfg["grad_chunk"] >= int(w)
    if cfg["grad_arena_bytes"] == 0:  # 8 warps need an 8-column chunk: chain32's workspace then exceeds the shared memory
        assert (name, w) == ("chain32", "8"), cfg
        with pytest.raises(RuntimeError, match=f"\\({DOJO_ENOMEM}\\)"):
            st.step_grad(np.tile(m.z0, (2, 1)))
    else:
        _gradient_parity(m, st, B, 23)
    st.close()
    # chain32: 48 environments, so that the 99 % quantile is not the largest of a handful of samples
    _compare_rollout(m, 48 if name == "chain32" else 24, 4, seed=9, scale=0.5, tol_median=1e-11)


def test_chunked_host_pointer_gradients():
    """chain32 (1.3 MB of Jacobians per environment): host-pointer dojo_step_grad in three chunks of the 128 MiB double buffer
    (the reuse of buffer 0 waits for its copy) and dojo_step_grad_contact in two chunks of its 192 MiB staging, bit-identical to
    the device-pointer path and to calls of one chunk each"""
    import torch
    from dojo_jl_b200.solver import BatchedStepper
    m = shape("chain32")
    ng, nu, nc = 12 * m.Nb, m.nu, 5 * m.Ni
    chunk = (128 << 20) // ((ng * ng + ng * nu) * 8)             # dojo_step_grad (dojo_b200.cu)
    chunk_c = (192 << 20) // ((ng * ng + ng * nu + ng * nc) * 8)  # dojo_step_grad_contact
    B, Bc = 2 * chunk + 7, chunk_c + 9
    Z, rng = _states(m, 16, 45)
    Z = Z[rng.integers(0, 16, max(B, Bc))]
    U = random_inputs(m, max(B, Bc), rng, 0.5)
    st = BatchedStepper(m, max(B, Bc))
    Zn, Fz, Fu, s, it = st.step_grad(Z[:B], U[:B])
    dZ, dU = torch.from_numpy(Z[:B]).cuda(), torch.from_numpy(U[:B]).cuda()
    dZn = torch.empty_like(dZ)
    dFz = torch.empty((B, ng, ng), dtype=torch.float64, device="cuda")
    dFu = torch.empty((B, nu, ng), dtype=torch.float64, device="cuda")
    st.step_grad_device(dZ.data_ptr(), dU.data_ptr(), dZn.data_ptr(), dFz.data_ptr(), dFu.data_ptr(), B)
    torch.cuda.synchronize()
    assert np.array_equal(dZn.cpu().numpy(), Zn)
    assert np.array_equal(dFz.cpu().numpy().transpose(0, 2, 1), Fz) and np.array_equal(dFu.cpu().numpy().transpose(0, 2, 1), Fu)
    for e0 in range(0, B, chunk):
        Zc, Fzc, Fuc, sc, itc = st.step_grad(Z[e0:e0 + chunk], U[e0:e0 + chunk])
        assert np.array_equal(Zc, Zn[e0:e0 + chunk]) and np.array_equal(Fzc, Fz[e0:e0 + chunk]) and np.array_equal(Fuc, Fu[e0:e0 + chunk])
        assert np.array_equal(sc, s[e0:e0 + chunk]) and np.array_equal(itc, it[e0:e0 + chunk])
    del dFz, dFu
    Zn2, Fz2, Fu2, Fc2, s2, it2 = st.step_grad_contact(Z[:Bc], U[:Bc])
    assert np.array_equal(Zn2, st.step(Z[:Bc], U[:Bc])[0])
    n = min(B, Bc)  # the same environments: the extra columns do not change the state / control gradients
    assert np.array_equal(Fz2[:n], Fz[:n]) and np.array_equal(Fu2[:n], Fu[:n])
    for e0 in range(0, Bc, chunk_c):
        e1 = min(Bc, e0 + chunk_c)
        _, Fzc, Fuc, Fcc, _, _ = st.step_grad_contact(Z[e0:e1], U[e0:e1])
        assert Fzc.shape[0] == Fcc.shape[0] == e1 - e0, (chunk_c, Bc, e0, Fzc.shape, Fcc.shape)
        bad = [e for e in range(e0, e1) if not (np.array_equal(Fzc[e - e0], Fz2[e]) and np.array_equal(Fcc[e - e0], Fc2[e]))]
        assert not bad, (chunk_c, Bc, e0, bad[:10])
    st.close()


@pytest.mark.parametrize("name", ["n33", "c33"])
def test_more_than_32_nodes_are_refused(name):
    from dojo_jl_b200.solver import BatchedStepper
    with pytest.raises(RuntimeError, match=f"\\({DOJO_EINVAL}\\).*up to 32 bodies / 32 joints / 32 contacts"):
        BatchedStepper(shape(name), 4)


def test_gradients_refused_when_the_workspace_does_not_fit():
    """big_nograd: the forward arena fits, the gradient workspace does not.  Steps and rollouts match the oracle; every gradient
    entry returns DOJO_ENOMEM with a message; the handle still steps correctly afterwards"""
    from dojo_jl_b200.solver import BatchedStepper
    from oracle.oracle import Oracle
    m = shape("big_nograd")
    B = 6
    Z, rng = _states(m, B, 51)
    U = random_inputs(m, B, rng, 0.5)
    st, o = BatchedStepper(m, B), Oracle(m)

    def check_step():
        Zn, s, it = st.step(Z, U)
        for e in range(B):
            zo, so, io = o.step(Z[e], U[e])
            assert (s[e], it[e]) == (so, io)
            assert so != 0 or np.abs(Zn[e] - zo).max() < 1e-6  # a :failed environment ends on an arbitrary iterate
        Zf, _ = st.rollout(Z, np.stack([U, U]), 2)
        assert np.array_equal(Zf, st.step(Zn, U)[0])

    check_step()
    for call in (lambda: st.step_grad(Z, U), lambda: st.step_grad_contact(Z, U),
                 lambda: st.minimal_gradients(st.maximal_to_minimal(Z), U)):
        with pytest.raises(RuntimeError, match=f"\\({DOJO_ENOMEM}\\): .+"):
            call()
    check_step()
    st.close()
