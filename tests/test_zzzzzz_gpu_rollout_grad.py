"""Trajectory Jacobians of a fused rollout on the H100 (run with -m gpu): dojo_rollout_grad is bit-identical to T sequential
dojo_step_grad calls and its trajectory to dojo_rollout's; the host- and device-pointer entries agree; the minimal-coordinate variant is
bit-identical to its per-step composition and its chained Jacobians match central differences of dojo_rollout; refused calls launch
nothing.  The CPU twin is tests/test_rollout_grad.py."""
import numpy as np
import pytest

import dojo_jl_b200 as dj
from conftest import jittered_states, random_inputs
from dojo_jl_b200 import capi

pytestmark = pytest.mark.gpu

DOJO_EINVAL, DOJO_ENOMEM = -1, -3
B, T = 64, 12


def _mech(name):
    if name == "block_linear":
        return dj.get_mechanism("block", contact_type="linear")
    return dj.get_mechanism(name)


def _start(m, B, T, seed):
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
    return Z, np.stack([random_inputs(m, B, rng, 0.5) for _ in range(T)])


def _same(got, ref, what):
    for k, (g, r) in enumerate(zip(got, ref)):
        assert g.shape == r.shape, (what, k, g.shape, r.shape)
        assert np.array_equal(g, r, equal_nan=True), f"{what}: output {k} differs (max |diff| {np.nanmax(np.abs(g - r))})"


@pytest.mark.parametrize("name", ("ant", "quadruped", "atlas", "block_linear"))
def test_equals_sequential_step_grad(name):
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech(name)
    st = BatchedStepper(m, B)
    Z0, U = _start(m, B, T, seed=31)
    got = st.rollout_grad(Z0, U, T)
    Z, seq = Z0, []
    for t in range(T):
        r = st.step_grad(Z, U[t])
        seq.append([a.copy() for a in r])
        Z = r[0]
    ref = (np.stack([Z0] + [r[0] for r in seq]),) + tuple(np.stack([r[k] for r in seq]) for k in range(1, 5))
    _same(got, ref, name)
    Zf, st_any, traj = st.rollout(Z0, U, T, record=True)
    assert np.array_equal(got[0][1:], traj) and np.array_equal(got[0][-1], Zf)
    assert np.array_equal(got[3].max(axis=0), st_any)
    st.close()


def test_host_and_device_pointers_agree():
    """the host entry runs the gradients in chunks of grad_chunk (= max_batch here) pairs after the rollout; the device entry overlaps
    the gradients of early steps with the rollout of later ones"""
    import torch
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech("ant")
    st = BatchedStepper(m, B)
    assert B * T > 2 * st.launch_config["grad_chunk"]  # several chunks, both staging buffers reused
    Z0, U = _start(m, B, T, seed=32)
    host = st.rollout_grad(Z0, U, T)
    ng, nu = st.ngrad, st.nu
    dZ = torch.empty((T + 1, B, st.nz), dtype=torch.float64, device="cuda")
    dZ[0] = torch.from_numpy(Z0).cuda()
    dU = torch.from_numpy(U).cuda()
    dFz = torch.empty((T, B, ng, ng), dtype=torch.float64, device="cuda")
    dFu = torch.empty((T, B, nu, ng), dtype=torch.float64, device="cuda")
    dst = torch.empty((T, B), dtype=torch.int32, device="cuda")
    dit = torch.empty((T, B), dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    st.rollout_grad_device(dZ.data_ptr(), dU.data_ptr(), dZ.data_ptr(), dFz.data_ptr(), dFu.data_ptr(), B, T, dstatus=dst.data_ptr(),
                           diters=dit.data_ptr(), stream=stream)
    torch.cuda.synchronize()
    dev = (dZ.cpu().numpy(), dFz.cpu().numpy().transpose(0, 1, 3, 2), dFu.cpu().numpy().transpose(0, 1, 3, 2), dst.cpu().numpy(), dit.cpu().numpy())
    _same(dev, host, "device vs host")
    # device pointers through the host-or-device entry, with Z0 in a buffer of its own
    dZ0 = torch.from_numpy(Z0).cuda()
    dZ.zero_()
    rc = st.L.dojo_rollout_grad(st.h, None, B, T, dZ0.data_ptr(), dU.data_ptr(), dZ.data_ptr(), dFz.data_ptr(), dFu.data_ptr(), None, None)
    assert rc == 0
    assert np.array_equal(dZ.cpu().numpy(), host[0]) and np.array_equal(dFz.cpu().numpy().transpose(0, 1, 3, 2), host[1])
    st.close()


def test_minimal_equals_per_step_composition():
    from dojo_jl_b200.solver import BatchedStepper
    for name in ("pendulum", "ant"):
        m = _mech(name)
        st = BatchedStepper(m, B)
        Z0, U = _start(m, B, T, seed=33)
        X0 = st.maximal_to_minimal(Z0)
        Xt, Gx, Gu, s, it = st.rollout_minimal_gradients(X0, U, T)
        traj, Fz, Fu, s2, it2 = st.rollout_grad(st.minimal_to_maximal(X0), U, T)
        assert np.array_equal(s, s2) and np.array_equal(it, it2)
        assert np.array_equal(Xt, np.stack([st.maximal_to_minimal(traj[t]) for t in range(T + 1)]))
        # the first step is one dojo_minimal_gradients call from X0 (the later ones re-enter maximal coordinates from X_traj[t])
        _same(st.minimal_gradients(X0, U[0]), (Xt[1], Gx[0], Gu[0], s[0], it[0]), name)
        # every step: M(z_{t+1}) Fz N(z_t), M(z_{t+1}) Fu from the map Jacobians of dojo_minimal_gradients' own kernel
        for t in (0, T // 2, T - 1):
            M, N = st.maximal_to_minimal_jacobian(traj[t + 1]), st.minimal_to_maximal_jacobian(traj[t])
            assert np.allclose(Gx[t], M @ Fz[t] @ N, rtol=1e-9, atol=1e-9), (name, t)
            assert np.allclose(Gu[t], M @ Fu[t], rtol=1e-9, atol=1e-9), (name, t)
        st.close()


def test_pendulum_chained_jacobian_matches_central_differences():
    from dojo_jl_b200.solver import BatchedStepper
    m = _mech("pendulum")
    assert m.Ni == 0
    st = BatchedStepper(m, 16)
    opts = capi.solver_options(rtol=1e-10, btol=1e-10)
    x0 = np.array([[0.7, -0.3]])
    U = np.full((T, 1, m.nu), 0.2)
    Xt, Gx, _, s, _ = st.rollout_minimal_gradients(x0, U, T, opts)
    assert (s == 0).all()
    J = np.eye(2)
    for t in range(T):
        J = Gx[t, 0] @ J
    eps = 1e-6
    X = np.concatenate([x0 + eps * np.eye(2), x0 - eps * np.eye(2)])
    Zf, s_any = st.rollout(st.minimal_to_maximal(X), np.repeat(U, 4, axis=1), T, opts)
    assert (s_any == 0).all()
    Xf = st.maximal_to_minimal(Zf)
    Jfd = ((Xf[:2] - Xf[2:]) / (2 * eps)).T
    assert np.linalg.norm(J - Jfd) <= 1e-6 * np.linalg.norm(J), (J, Jfd)


def test_refusals():
    from dojo_jl_b200.solver import BatchedStepper
    from test_shape_boundaries import shape
    m = _mech("ant")
    st = BatchedStepper(m, 8)
    Z0, U = _start(m, 9, 2, seed=34)
    X4 = st.maximal_to_minimal(Z0[:4])
    n = st.launch_count
    with pytest.raises(RuntimeError, match=f"\\({DOJO_EINVAL}\\): .+"):
        st.rollout_grad(Z0, U, 2)  # B = 9 > max_batch
    with pytest.raises(RuntimeError, match=f"\\({DOJO_EINVAL}\\): .+"):
        st.rollout_grad(Z0[:4], U[:0, :4], 0)
    with pytest.raises(RuntimeError, match=f"\\({DOJO_EINVAL}\\): .+"):
        st.rollout_minimal_gradients(X4, U[:0, :4], 0)
    assert st.launch_count == n
    st.close()
    big = BatchedStepper(shape("big_nograd"), 4)
    mb = big.mech
    Zb = np.tile(mb.z0, (2, 1))
    Xb = big.maximal_to_minimal(Zb)
    n = big.launch_count
    for call in (lambda: big.rollout_grad(Zb, None, 3), lambda: big.rollout_minimal_gradients(Xb, None, 3)):
        with pytest.raises(RuntimeError, match=f"\\({DOJO_ENOMEM}\\): .+"):
            call()
    assert big.launch_count == n
    big.close()
