"""Timing of reverse mode through a closed-loop rollout: dojo_rollout_feedback_tape + dojo_rollout_feedback_vjp.

    python tools/feedback_vjp_time.py [--work ant:4096:100 atlas:1024:100] [--repeats 7] [--warmup 1]

Per workload, from bench.py's seeded batch after its roll-in (synthetic_batch, random_inputs, WORKLOADS) and a seeded law -- K shared by
the steps, small random gains per environment, x_ref the batch's starting minimal state -- each call timed alone with CUDA events, arms
alternated within every repeat:
  fb        dojo_rollout_feedback_async (the closed-loop rollout, trajectory and applied inputs recorded);
  fb_tape   dojo_rollout_feedback_tape_async (the same rollout, recorded for the adjoint);
  fb_vjp    dojo_rollout_feedback_vjp_async (one adjoint pass through the closed loop, random cotangents on z_t, x_t and u_t, every law
            gradient written);
  tape_vjp  dojo_rollout_tape_async + dojo_rollout_vjp_async driven by the same applied inputs (the open loop's reverse mode).
Before timing, the tape's trajectory is compared with the closed-loop rollout's and with the open-loop tape's, and the closed-loop
rollout with a repeat of itself: where the forward kernel is not reproducible from run to run (atlas, whose solves end :failed on ~9%
of the pairs), the first comparison cannot hold either.  Prints medians and interquartile ranges, the card, its power limit and SM clock, and one JSON line.
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
    from dojo_jl_b200 import capi
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism(name)
    w = bench.WORKLOADS[name]
    opts = capi.solver_options()
    st = BatchedStepper(mech, B)
    nz, nu, ng, nres, nx = st.nz, st.nu, st.ngrad, st.nres, 2 * st.nu
    Z0, rng = bench.synthetic_batch(mech, B, 0xD0D0 + 1, name)
    U = torch.from_numpy(bench.random_inputs(mech, rng, max(w["rollin"], 1), B, bench.SCALE.get(name, 1.0))).cuda()
    Za, Zb = torch.from_numpy(Z0).cuda(), torch.empty((B, nz), dtype=torch.float64, device="cuda")
    for t in range(w["rollin"]):
        st.step_device(Za.data_ptr(), U[t].data_ptr(), Zb.data_ptr(), B, opts)
        Za, Zb = Zb, Za
    f64, i32 = dict(dtype=torch.float64, device="cuda"), dict(dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    X0 = torch.from_numpy(st.maximal_to_minimal(Za.cpu().numpy())).cuda()
    g = np.random.default_rng(11)
    K = torch.from_numpy(np.ascontiguousarray(g.normal(0.0, 0.05, (1, B, nx, nu)))).cuda()  # column-major [nu x 2nu] per entry
    xr = X0.reshape(1, B, nx).contiguous()
    gen = torch.Generator(device="cuda").manual_seed(7)
    gZ, gX, gU = (torch.randn(sh, generator=gen, **f64) for sh in ((T + 1, B, ng), (T + 1, B, nx), (T, B, nu)))
    b = dict(traj=torch.empty((T + 1, B, nz), **f64), X=torch.empty((T + 1, B, nx), **f64), Ua=torch.empty((T, B, nu), **f64),
             tape=torch.empty((T, B, nres), **f64), st=torch.empty((T, B), **i32), gZ0=torch.empty((B, ng), **f64), gK=torch.empty((1, B, nx, nu), **f64),
             gxr=torch.empty((1, B, nx), **f64), gur=torch.empty((1, B, nu), **f64), vst=torch.empty(B, **i32), Zf=torch.empty((B, nz), **f64),
             ftraj=torch.empty((T, B, nz), **f64), fUa=torch.empty((T, B, nu), **f64), fst=torch.empty(B, **i32),
             otraj=torch.empty((T + 1, B, nz), **f64), otape=torch.empty((T, B, nres), **f64), ost=torch.empty((T, B), **i32),
             ogZ0=torch.empty((B, ng), **f64), ogU=torch.empty((T, B, nu), **f64))
    p = lambda k: b[k].data_ptr()  # noqa: E731

    def fb():
        st.rollout_feedback_device(Za.data_ptr(), p("Zf"), B, T, K.data_ptr(), steps=1, envs=B, dx_ref=xr.data_ptr(), dtraj=p("ftraj"),
                                   dU_applied=p("fUa"), dstatus=p("fst"), opts=opts, stream=s)

    def fb_tape():
        st.rollout_feedback_tape_device(Za.data_ptr(), p("traj"), p("X"), p("Ua"), p("tape"), B, T, K.data_ptr(), steps=1, envs=B, dx_ref=xr.data_ptr(),
                                        dstatus=p("st"), opts=opts, stream=s)

    def fb_vjp():
        st.rollout_feedback_vjp_device(p("traj"), p("X"), p("Ua"), p("tape"), p("gZ0"), B, T, K.data_ptr(), steps=1, envs=B, dx_ref=xr.data_ptr(),
                                       dgZ=gZ.data_ptr(), dgX=gX.data_ptr(), dgU=gU.data_ptr(), dgK=p("gK"), dgx_ref=p("gxr"), dgu_ref=p("gur"),
                                       dstatus=p("vst"), stream=s)

    def tape_vjp():
        st.rollout_tape_device(Za.data_ptr(), p("Ua"), p("otraj"), p("otape"), B, T, opts, dstatus=p("ost"), stream=s)
        st.rollout_vjp_device(p("otraj"), p("Ua"), p("otape"), gZ.data_ptr(), p("ogZ0"), B, T, dgU=p("ogU"), stream=s)

    for _ in range(warmup + 1):
        fb(); fb_tape(); fb_vjp(); tape_vjp()
    torch.cuda.synchronize()
    same = bool(torch.equal(b["traj"][1:], b["ftraj"]) and torch.equal(b["Ua"], b["fUa"]) and torch.equal(b["traj"], b["otraj"])
                and torch.equal(b["tape"], b["otape"]))
    ftraj0 = b["ftraj"].clone()
    fb()
    torch.cuda.synchronize()
    repeat = bool(torch.equal(b["ftraj"], ftraj0))  # the closed-loop rollout against itself: the floor of the comparison above
    finite = bool(torch.isfinite(b["gZ0"]).all() and torch.isfinite(b["gK"]).all())
    arms = {"fb": fb, "fb_tape": fb_tape, "fb_vjp": fb_vjp, "tape_vjp": tape_vjp}
    times = {k: [] for k in arms}
    order = list(arms)
    for r in range(repeats):
        for k in order[r % len(order):] + order[:r % len(order)]:
            times[k].append(_timed(arms[k]))
    res = {k: _q(v) for k, v in times.items()}
    print(f"{name}: B = {B}, T = {T}; tape equals both rollouts bit for bit: {same} (the closed-loop rollout equals itself when "
          f"repeated: {repeat}); adjoint finite: {finite}; "
          f"adjoint status 3 in {int((b['vst'] != 0).sum())} environments")
    for k in arms:
        print(f"  {k:9s} {res[k][0]:10.2f} ms  (IQR {res[k][1]:.2f})")
    return {"mech": name, "B": B, "T": T, "ms": {k: res[k][0] for k in arms}, "iqr_ms": {k: res[k][1] for k in arms}, "tape_bitwise": same, "fb_repeat_bitwise": repeat,
            "finite": finite}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--work", nargs="+", default=["ant:4096:100", "atlas:1024:100"])
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    card = _card()
    print("card (name, power limit, max SM clock, SM clock):", card)
    rows = []
    for wk in a.work:
        name, B, T = wk.split(":")
        rows.append(run(name, int(B), int(T), a.repeats, a.warmup))
    print(json.dumps({"card": card, "results": rows}))


if __name__ == "__main__":
    main()
