"""Timing of reverse mode through a rollout: dojo_rollout_tape + dojo_rollout_vjp against the Jacobians of dojo_rollout_grad.

    python tools/rollout_vjp_time.py [--work ant:4096:100 atlas:1024:100] [--jac-batch 2048 256] [--repeats 7] [--warmup 1]

Per workload, from bench.py's seeded batch after its roll-in (synthetic_batch, random_inputs, WORKLOADS) and T seeded inputs, each call
timed alone with CUDA events, arms alternated within every repeat:
  roll   dojo_rollout_async (the plain rollout, trajectory recorded);
  tape   dojo_rollout_tape_async (the same rollout keeping every step's final iterate);
  vjp    dojo_rollout_vjp_async (one adjoint pass over the tape, a random cotangent on every slab).
At full size the Jacobians do not fit on the device, so the Jacobian route is timed at the smaller batch --jac-batch, with the VJP at
that batch too:
  jac    dojo_rollout_grad_async, then the contraction lambda_t = Fz' lambda_{t+1} + gZ[t], gU[t] = Fu' lambda_{t+1} as torch bmm per step;
  vjp_b  tape + vjp at the same batch.
Before timing, the jac and vjp_b results are compared (largest difference relative to the largest entry, and the largest difference
of the two trajectories).  Prints medians and
interquartile ranges, bytes per (environment, step) pair of both routes from the shapes, the card, its power limit and SM clock, and
one JSON line.
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


def run(name, B, T, Bj, repeats, warmup):
    import torch
    import bench
    import dojo_jl_b200 as dj
    from dojo_jl_b200 import capi
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism(name)
    w = bench.WORKLOADS[name]
    opts = capi.solver_options()
    st = BatchedStepper(mech, B)
    nz, nu, ng, nres = st.nz, st.nu, st.ngrad, st.nres
    Z0, rng = bench.synthetic_batch(mech, B, 0xD0D0 + 1, name)
    U = torch.from_numpy(bench.random_inputs(mech, rng, w["rollin"] + T, B, bench.SCALE.get(name, 1.0))).cuda()
    Za, Zb = torch.from_numpy(Z0).cuda(), torch.empty((B, nz), dtype=torch.float64, device="cuda")
    for t in range(w["rollin"]):
        st.step_device(Za.data_ptr(), U[t].data_ptr(), Zb.data_ptr(), B, opts)
        Za, Zb = Zb, Za
    U = U[w["rollin"]:].contiguous()
    f64, i32 = dict(dtype=torch.float64, device="cuda"), dict(dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    gen = torch.Generator(device="cuda").manual_seed(7)
    gZ = torch.randn((T + 1, B, ng), generator=gen, **f64)

    def buffers(b):
        traj = torch.empty((T + 1, b, nz), **f64)
        traj[0] = Za[:b]
        return dict(traj=traj, tape=torch.empty((T, b, nres), **f64), st=torch.empty((T, b), **i32), gZ0=torch.empty((b, ng), **f64),
                    gU=torch.empty((T, b, nu), **f64), vst=torch.empty(b, **i32), Zf=torch.empty((b, nz), **f64))

    full = buffers(B)
    Ub = lambda b: U[:, :b].contiguous()  # noqa: E731
    Uf = U

    def roll():
        st.rollout_device(full["traj"][0].data_ptr(), Uf.data_ptr(), full["Zf"].data_ptr(), B, T, opts, dtraj=full["traj"][1].data_ptr(), stream=s)

    def tape(bb=full, b=B, u=Uf):
        st.rollout_tape_device(bb["traj"][0].data_ptr(), u.data_ptr(), bb["traj"].data_ptr(), bb["tape"].data_ptr(), b, T, opts,
                               dstatus=bb["st"].data_ptr(), stream=s)

    def vjp(bb=full, b=B, u=Uf, g=gZ):
        st.rollout_vjp_device(bb["traj"].data_ptr(), u.data_ptr(), bb["tape"].data_ptr(), g.data_ptr(), bb["gZ0"].data_ptr(), b, T,
                              dgU=bb["gU"].data_ptr(), dstatus=bb["vst"].data_ptr(), stream=s)

    # the Jacobian route at the batch that fits
    small, us, gs = buffers(Bj), Ub(Bj), gZ[:, :Bj].contiguous()
    Fz, Fu = torch.empty((T, Bj, ng, ng), **f64), torch.empty((T, Bj, nu, ng), **f64)
    jtraj, jst = torch.empty((T + 1, Bj, nz), **f64), torch.empty((T, Bj), **i32)
    jtraj[0] = Za[:Bj]
    out = {}

    def jac():
        st.rollout_grad_device(jtraj[0].data_ptr(), us.data_ptr(), jtraj.data_ptr(), Fz.data_ptr(), Fu.data_ptr(), Bj, T, opts, dstatus=jst.data_ptr(),
                               stream=s)
        lam = gs[T].unsqueeze(-1)
        gU = torch.empty((T, Bj, nu), **f64)
        for t in range(T - 1, -1, -1):  # Fz[t, e] is column-major: its memory is Fz', so Fz' lambda is the row-major product
            gU[t] = torch.bmm(Fu[t], lam).squeeze(-1)
            lam = torch.bmm(Fz[t], lam) + gs[t].unsqueeze(-1)
        out["gZ0"], out["gU"] = lam.squeeze(-1), gU

    def vjp_b():
        tape(small, Bj, us)
        vjp(small, Bj, us, gs)

    for _ in range(warmup + 1):
        roll(); tape(); vjp(); jac(); vjp_b()
    torch.cuda.synchronize()
    diff = max(float((out["gZ0"] - small["gZ0"]).abs().max() / out["gZ0"].abs().max()),
               float((out["gU"] - small["gU"]).abs().max() / out["gU"].abs().max()) if nu else 0.0)
    traj_diff = float((jtraj - small["traj"]).abs().max())  # reported: the two routes' rollouts, each timed as it runs
    arms = {"roll": roll, "tape": tape, "vjp": vjp, "jac": jac, "vjp_b": vjp_b}
    times = {k: [] for k in arms}
    order = list(arms)
    for r in range(repeats):
        for k in order[r % len(order):] + order[:r % len(order)]:
            times[k].append(_timed(arms[k]))
    res = {k: _q(v) for k, v in times.items()}
    bytes_vjp = 8 * (nz + nres + ng + nu)        # trajectory slab, tape, cotangent slab, input gradient per pair
    bytes_jac = 8 * (ng * ng + ng * nu + nz)     # Fz, Fu and the trajectory slab per pair
    print(f"{name}: B = {B}, T = {T} (Jacobian route at B = {Bj}); relative difference jac vs vjp {diff:.1e}, largest trajectory "
          f"difference between the two routes {traj_diff:.1e}")
    for k in arms:
        print(f"  {k:6s} {res[k][0]:10.2f} ms  (IQR {res[k][1]:.2f})")
    print(f"  bytes per pair: vjp route {bytes_vjp}, Jacobian route {bytes_jac}")
    return {"mech": name, "B": B, "T": T, "B_jac": Bj, "ms": {k: res[k][0] for k in arms}, "iqr_ms": {k: res[k][1] for k in arms},
            "bytes_per_pair_vjp": bytes_vjp, "bytes_per_pair_jac": bytes_jac, "rel_diff_jac_vs_vjp": diff, "traj_diff": traj_diff}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--work", nargs="+", default=["ant:4096:100", "atlas:1024:100"])
    p.add_argument("--jac-batch", nargs="+", type=int, default=[2048, 256])
    p.add_argument("--repeats", type=int, default=7)
    p.add_argument("--warmup", type=int, default=1)
    a = p.parse_args()
    card = _card()
    print("card (name, power limit, max SM clock, SM clock):", card)
    rows = []
    for wk, bj in zip(a.work, a.jac_batch):
        name, B, T = wk.split(":")
        rows.append(run(name, int(B), int(T), bj, a.repeats, a.warmup))
    print(json.dumps({"card": card, "results": rows}))


if __name__ == "__main__":
    main()
