"""Timing of the Riccati backward pass: dojo_lqr_backward_async against the same recursion as per-step torch ops, and against the
rollout with Jacobians that feeds it.

    python tools/lqr_backward_time.py [--mech ant] [--batch 4096] [--steps 100] [--repeats 5]

From bench.py's seeded batch (synthetic_batch, random_inputs), one dojo_rollout_minimal_gradients gives X_traj, Gx and Gu on the device
(the floating base inactive, as an iLQR of the mechanism would have it).  Cost: Q = I, R = 0.1 I, Q_final = 10 I, goal 0, mu = 1e-6.
  kernel  one dojo_lqr_backward_async (dojo_lqr.cuh: one CTA per environment, all T steps in one launch);
  torch   the recursion a user writes without it: per step batched bmm / cholesky / cholesky_solve over the B environments;
  rollmg  one dojo_rollout_minimal_gradients at the same size (device pointers), for the share of an iLQR iteration the pass is.
Before timing, K, k and dV of kernel and torch are compared on the environments whose Cholesky succeeded (max relative difference
printed; the two round differently).  Each repeat
runs the arms in a rotating order, each call timed alone with CUDA events.  Prints per arm the median and interquartile range, the
bytes of Gx / Gu read and the flops of the recursion's products counted from shapes (not measured) over the kernel's median time, the
card and its power limit, and one JSON line.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _q(x):
    q1, med, q3 = np.percentile(np.asarray(x, float), [25, 50, 75])
    return float(med), float(q3 - q1)


def _card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still printed; the card is then reported unknown
        return f"unknown ({e})"


def counts(nu, na, B, T):
    """(bytes of Gx / Gu read, flops of the recursion's products) from shapes: PA, A'PA (nx^3 each), PB, B'PA (nx^2 na), B'PB (nx na^2),
    Quu K, K'W, Qux'K (na^2 nx, 2 nx^2 na), Cholesky and solves (na^3 / 3, 2 na^2 (nx + 1)); a multiply-add is two flops"""
    nx = 2 * nu
    fma = 2 * nx ** 3 + 2 * nx * nx * na + nx * na * na + na * na * nx + 2 * nx * nx * na + na ** 3 / 6 + na * na * (nx + 1)
    return 8.0 * (nx * nx + nx * nu) * B * T, 2.0 * fma * B * T


def torch_backward(torch, X, Gxc, Guc, act, Q, R, Qf, mu):
    """the recursion of dojo_lqr.cuh as per-step batched torch ops; X [T+1, B, nx], Gxc / Guc column-major per pair"""
    T, B, nx = Gxc.shape[0], Gxc.shape[1], Gxc.shape[2]
    nu = Guc.shape[2]
    K = torch.zeros((T, B, nu, nx), dtype=X.dtype, device=X.device)
    k = torch.zeros((T, B, nu), dtype=X.dtype, device=X.device)
    dV = torch.zeros((B, 2), dtype=X.dtype, device=X.device)
    Ra = R[act][:, act]
    muI = mu[:, None, None] * torch.eye(len(act), dtype=X.dtype, device=X.device)
    P = Qf.expand(B, nx, nx).clone()
    p = X[T] @ Qf.T
    for t in range(T - 1, -1, -1):
        A = Gxc[t].transpose(1, 2)
        Bu = Guc[t][:, act, :].transpose(1, 2)
        PA, PB = torch.bmm(P, A), torch.bmm(P, Bu)
        Qx = X[t] @ Q.T + torch.bmm(A.transpose(1, 2), p[:, :, None])[:, :, 0]
        Qu = torch.bmm(Bu.transpose(1, 2), p[:, :, None])[:, :, 0]
        Qxx = Q + torch.bmm(A.transpose(1, 2), PA)
        Quu = Ra + torch.bmm(Bu.transpose(1, 2), PB)
        Qux = torch.bmm(Bu.transpose(1, 2), PA)
        L, _ = torch.linalg.cholesky_ex(Quu + muI)
        Y = torch.cholesky_solve(torch.cat([Qux, -Qu[:, :, None]], 2), L)
        Ka, ka = Y[:, :, :nx], Y[:, :, nx]
        W = torch.bmm(Quu, Ka) - Qux
        P = Qxx + torch.bmm(Ka.transpose(1, 2), W) - torch.bmm(Qux.transpose(1, 2), Ka)
        P = 0.5 * (P + P.transpose(1, 2))
        qk = torch.bmm(Quu, ka[:, :, None])[:, :, 0]
        p = Qx - torch.bmm(Ka.transpose(1, 2), (qk + Qu)[:, :, None])[:, :, 0] + torch.bmm(Qux.transpose(1, 2), ka[:, :, None])[:, :, 0]
        dV[:, 0] += (ka * Qu).sum(1)
        dV[:, 1] += 0.5 * (ka * qk).sum(1)
        K[t][:, act] = Ka
        k[t][:, act] = ka
    return K, k, dV


def run(name, B, T, repeats):
    import torch
    import bench
    import dojo_jl_b200 as dj
    from dojo_jl_b200 import capi
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism(name)
    st = BatchedStepper(mech, B)
    nu, nx, nz = st.nu, 2 * st.nu, st.nz
    Z0, rng = bench.synthetic_batch(mech, B, 0xD0D0 + 1, name)
    act_mask = np.ones(nu, dtype=np.int32)
    off = 0
    for j in mech.joints:
        if j.nimpulses == 0:
            act_mask[off:off + j.input_dimension] = 0
        off += j.input_dimension
    act = np.flatnonzero(act_mask)
    f64 = dict(dtype=torch.float64, device="cuda")
    U = torch.from_numpy(np.ascontiguousarray(bench.random_inputs(mech, rng, T, B, bench.SCALE.get(name, 1.0)))).cuda()
    X0 = torch.from_numpy(st.maximal_to_minimal(Z0)).cuda()
    X = torch.empty((T + 1, B, nx), **f64)
    Gx, Gu = torch.empty((T, B, nx, nx), **f64), torch.empty((T, B, nu, nx), **f64)  # column-major per pair
    stat, iters = torch.empty((T, B), dtype=torch.int32, device="cuda"), torch.empty((T, B), dtype=torch.int32, device="cuda")
    o = capi.solver_options()
    vp = lambda t: C.c_void_p(t.data_ptr())

    def rollmg():
        rc = st.L.dojo_rollout_minimal_gradients(st.h, C.byref(o), B, T, vp(X0), vp(U), vp(X), vp(Gx), vp(Gu), vp(stat), vp(iters))
        assert rc == 0, st.L.dojo_last_error(st.h)

    rollmg()
    torch.cuda.synchronize()
    Q, R, Qf = torch.eye(nx, **f64), 0.1 * torch.eye(nu, **f64), 10.0 * torch.eye(nx, **f64)
    mu = torch.full((B,), 1e-6, **f64)
    K, k, dV = torch.empty((T, B, nx, nu), **f64), torch.empty((T, B, nu), **f64), torch.empty((B, 2), **f64)
    status = torch.empty((B,), dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def kernel():
        st.lqr_backward_device(B, T, X.data_ptr(), Gx.data_ptr(), Gu.data_ptr(), K.data_ptr(), k.data_ptr(), Q.data_ptr(), R.data_ptr(),
                               Qf.data_ptr(), dmu=mu.data_ptr(), active=act_mask, ddV=dV.data_ptr(), dstatus=status.data_ptr(), stream=stream)

    act_t = torch.from_numpy(act).cuda()
    tout = {}

    def torch_arm():
        tout["r"] = torch_backward(torch, X, Gx, Gu, act_t, Q, R, Qf, mu)

    kernel()
    torch_arm()
    torch.cuda.synchronize()
    Kt, kt, dVt = tout["r"]
    ok = status == 0
    rel = lambda a, b: float((a - b).abs().max() / b.abs().max().clamp(min=1.0))
    check = dict(failed=int((~ok).sum()), K=rel(K.transpose(2, 3)[:, ok], Kt[:, ok]), k=rel(k[:, ok], kt[:, ok]), dV=rel(dV[ok], dVt[ok]))
    print(f"{name} B={B} T={T}: kernel vs torch max relative difference K {check['K']:.1e} k {check['k']:.1e} dV {check['dV']:.1e}, "
          f"failed Cholesky {check['failed']}", flush=True)
    # 100 steps of the recursion on these Jacobians amplify the different rounding of the two arms to about 1e-6 (ant) / 1e-5 (atlas)
    # relative; the recursion itself is checked to 1e-9 against numpy at T = 12 (tests/test_zzzzzzzz_gpu_lqr.py)
    assert max(check["K"], check["k"], check["dV"]) < 1e-4, check
    arms = {"kernel": kernel, "torch": torch_arm, "rollmg": rollmg}
    times = {a: [] for a in arms}
    names = list(arms)
    for r in range(repeats):
        for a in names[r % 3:] + names[: r % 3]:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            arms[a]()
            e1.record()
            torch.cuda.synchronize()
            times[a].append(e0.elapsed_time(e1) * 1e-3)
    by, fl = counts(nu, len(act), B, T)
    out = {"mech": name, "B": B, "T": T, "card": _card(), "check": check, "bytes_GxGu": by, "flops": fl}
    for a in names:
        med, iqr = _q(times[a])
        out[a + "_s"], out[a + "_iqr_s"] = med, iqr
        print(f"  {a:7s} median {med * 1e3:9.2f} ms  IQR {iqr * 1e3:7.2f} ms", flush=True)
    out["kernel_GBps"], out["kernel_GFLOPs"] = by / out["kernel_s"] / 1e9, fl / out["kernel_s"] / 1e9
    out["torch_over_kernel"] = out["torch_s"] / out["kernel_s"]
    out["kernel_share_of_iteration"] = out["kernel_s"] / (out["kernel_s"] + out["rollmg_s"])
    print(f"  kernel: {by / 1e9:.2f} GB of Gx/Gu at {out['kernel_GBps']:.0f} GB/s, {fl:.2e} flops at {out['kernel_GFLOPs']:.0f} GFLOP/s (counted "
          f"from shapes); torch / kernel = {out['torch_over_kernel']:.2f}; card: {out['card']}", flush=True)
    st.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mech", default="ant")
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    print(json.dumps(run(a.mech, a.batch, a.steps, a.repeats)))


if __name__ == "__main__":
    main()
