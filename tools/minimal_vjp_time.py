"""Timing of reverse mode in minimal coordinates: the adjoints of the coordinate maps next to the rollout tape and adjoint they compose with.

    python tools/minimal_vjp_time.py [--work ant:4096:100 atlas:1024:100] [--repeats 5] [--warmup 1]

Per workload, from bench.py's seeded batch after its roll-in (synthetic_batch, random_inputs, WORKLOADS), each call timed alone with CUDA
events, arms alternated within every repeat:
  tape       dojo_rollout_tape_async (B environments, T steps);
  vjp        dojo_rollout_vjp_async (one adjoint pass, cotangents on every slab);
  mT         dojo_maximal_to_minimal_vjp_async over the B (T+1) slabs of the trajectory in one call (gZ[t] = M(z_t)' gX[t]);
  nT         dojo_minimal_to_maximal_vjp_async over the B start states (gX0 = N(z_0)' lambda_0);
  dense      the same M' products the dense way: dojo_maximal_to_minimal_jacobian_async per slab plus a torch bmm;
  ag_min     autograd.rollout_minimal forward + backward (loss: a fixed random projection of X_traj);
  ag_max     autograd.rollout forward + backward from the same maximal start (loss: a fixed random projection of Z_traj).
Before timing, mT is compared with the dense route (largest difference relative to the largest entry).  Prints medians and interquartile
ranges, the card, its power limit and SM clocks, and one JSON line.
"""
import argparse
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
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still printed; the card is then reported unknown
        return f"unknown ({e})"


def _timed(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def run(name, B, T, repeats, warmup):
    import torch
    import bench
    import dojo_jl_b200 as dj
    from dojo_jl_b200 import autograd, capi
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism(name)
    w = bench.WORKLOADS[name]
    opts = capi.solver_options()
    st = BatchedStepper(mech, B)
    nz, nu, ng, nres, nx = st.nz, st.nu, st.ngrad, st.nres, 2 * st.nu
    Z0, rng = bench.synthetic_batch(mech, B, 0xD0D0 + 1, name)
    Ur = torch.from_numpy(bench.random_inputs(mech, rng, max(w["rollin"], 1), B, bench.SCALE.get(name, 1.0))).cuda()
    Za, Zb = torch.from_numpy(Z0).cuda(), torch.empty((B, nz), dtype=torch.float64, device="cuda")
    for t in range(w["rollin"]):
        st.step_device(Za.data_ptr(), Ur[t].data_ptr(), Zb.data_ptr(), B, opts)
        Za, Zb = Zb, Za
    f64 = dict(dtype=torch.float64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    U = torch.from_numpy(bench.random_inputs(mech, rng, T, B, bench.SCALE.get(name, 1.0))).cuda().contiguous()
    X0 = torch.empty((B, nx), **f64)
    st.maximal_to_minimal_device(Za.data_ptr(), X0.data_ptr(), B, stream=s)
    Zs = torch.empty((B, nz), **f64)
    st.minimal_to_maximal_device(X0.data_ptr(), Zs.data_ptr(), B, stream=s)  # the start autograd.rollout_minimal maps to
    gen = torch.Generator(device="cuda").manual_seed(7)
    gX, gZr = torch.randn((T + 1, B, nx), generator=gen, **f64), torch.randn((T + 1, B, nz), generator=gen, **f64)
    traj, tape = torch.empty((T + 1, B, nz), **f64), torch.empty((T, B, nres), **f64)
    gZ, gZd, gZ0, gU, gX0 = (torch.empty(sh, **f64) for sh in ((T + 1, B, ng), (T + 1, B, ng), (B, ng), (T, B, nu), (B, nx)))
    J = torch.empty((B, ng, nx), **f64)  # column-major [2nu x 12Nb] per environment

    def tape_():
        st.rollout_tape_device(Zs.data_ptr(), U.data_ptr(), traj.data_ptr(), tape.data_ptr(), B, T, opts, stream=s)

    def vjp():
        st.rollout_vjp_device(traj.data_ptr(), U.data_ptr(), tape.data_ptr(), gZ.data_ptr(), gZ0.data_ptr(), B, T, dgU=gU.data_ptr(), stream=s)

    def mT():
        st.maximal_to_minimal_vjp_device(traj.data_ptr(), gX.data_ptr(), gZ.data_ptr(), B * (T + 1), stream=s)

    def nT():
        st.minimal_to_maximal_vjp_device(traj.data_ptr(), gZ0.data_ptr(), gX0.data_ptr(), B, stream=s)

    def dense():
        for t in range(T + 1):
            st.maximal_to_minimal_jacobian_device(traj[t].data_ptr(), J.data_ptr(), B, stream=s)
            torch.bmm(J, gX[t].unsqueeze(2), out=gZd[t].unsqueeze(2))

    Xm0 = X0.clone().requires_grad_(True)
    Zm0 = Zs.clone().requires_grad_(True)
    Ua = U.clone().requires_grad_(True)

    def ag_min():
        Xt, _ = autograd.rollout_minimal(mech, Xm0, Ua, opts)
        (Xt * gX).sum().backward()

    def ag_max():
        Zt, _ = autograd.rollout(mech, Zm0, Ua, opts)
        (Zt * gZr).sum().backward()

    arms = {"tape": tape_, "vjp": vjp, "mT": mT, "nT": nT, "dense": dense, "ag_min": ag_min, "ag_max": ag_max}
    tape_()
    for _ in range(warmup + 1):
        for f in arms.values():
            f()
    torch.cuda.synchronize()
    mT(); dense()
    torch.cuda.synchronize()
    dense_diff = float((gZ - gZd).abs().max() / gZd.abs().max())
    times = {k: [] for k in arms}
    order = list(arms)
    for r in range(repeats):
        for k in order[r % len(order):] + order[:r % len(order)]:
            times[k].append(_timed(arms[k]))
    res = {k: _q(v) for k, v in times.items()}
    bytes_mT = B * (T + 1) * 8 * (nz + nx + ng)
    print(f"{name}: B = {B}, T = {T}, n = B (T+1) = {B * (T + 1)} slabs; M' against the dense route: {dense_diff:.1e} of the largest entry; "
          f"M' moves {bytes_mT / 1e6:.0f} MB ({bytes_mT / (B * (T + 1)):.0f} B per state)")
    for k in arms:
        print(f"  {k:7s} {res[k][0]:10.3f} ms  (IQR {res[k][1]:.3f})")
    print(f"  mT / vjp = {res['mT'][0] / res['vjp'][0]:.3f};  mT achieved {bytes_mT / res['mT'][0] / 1e6:.0f} GB/s")
    return {"mech": name, "B": B, "T": T, "ms": {k: res[k][0] for k in arms}, "iqr_ms": {k: res[k][1] for k in arms}, "mT_vs_dense": dense_diff,
            "mT_bytes": bytes_mT}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--work", nargs="+", default=["ant:4096:100", "atlas:1024:100"])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    card = _card()
    print("card (name, power limit, max SM clock, SM clock):", card)
    rows = []
    for wk in a.work:
        name, B, T = wk.split(":")
        rows.append(run(name, int(B), int(T), a.repeats, a.warmup))
    print("card after the runs:", _card())
    print(json.dumps({"card": card, "results": rows}))


if __name__ == "__main__":
    main()
