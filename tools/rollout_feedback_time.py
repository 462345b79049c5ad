"""Timing of the closed-loop rollout: dojo_rollout_feedback_async against the open-loop rollout and the per-step composition.

    python tools/rollout_feedback_time.py [--mech ant] [--batch 4096] [--steps 20] [--repeats 10] [--warmup 2]

From bench.py's seeded batch after its roll-in (synthetic_batch, random_inputs, WORKLOADS), a linear law u = -K (x - x_ref) with
x_ref = the minimal state after the roll-in and K a seeded [nu x 2nu] matrix of small gains, the same for every environment:
  fb       one dojo_rollout_feedback_async (the FB kernel: generic in the warp count), recording U_applied;
  roll     one dojo_rollout_async driven by the recorded U_applied, with the forward kernel dojo_create picks (for ant: the SMALL one);
  rollgen  the same with the generic forward kernel (a second handle created under DOJO_B200_GENERIC_STEP=1);
  perstep  what a caller composes without the FB kernel: per step dojo_maximal_to_minimal_async, the law as torch ops, dojo_step_async.
fb - rollgen is the cost of the feedback stage, rollgen - roll the difference between the kernel variants.  Before timing, the final states
of fb, roll and rollgen are checked to be bit-identical (perstep rounds the law differently and is not compared).  Each repeat runs the
arms in a rotating order, each call timed alone with CUDA events.  Prints the median and interquartile range per arm, the medians of the
per-repeat ratios, the card and its power limit, and one JSON line.
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
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still printed; the card is then reported unknown
        return f"unknown ({e})"


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
    os.environ["DOJO_B200_GENERIC_STEP"] = "1"
    try:
        gen = BatchedStepper(mech, B)
    finally:
        del os.environ["DOJO_B200_GENERIC_STEP"]
    nz, nu = st.nz, st.nu
    Z0, rng = bench.synthetic_batch(mech, B, 0xD0D0 + 1, name)
    U = torch.from_numpy(bench.random_inputs(mech, rng, max(w["rollin"], 1), B, bench.SCALE.get(name, 1.0))).cuda()
    f64, i32 = dict(dtype=torch.float64, device="cuda"), dict(dtype=torch.int32, device="cuda")
    Za, Zb = torch.from_numpy(Z0).cuda(), torch.empty((B, nz), **f64)
    for t in range(w["rollin"]):
        st.step_device(Za.data_ptr(), U[t].data_ptr(), Zb.data_ptr(), B, opts)
        Za, Zb = Zb, Za
    torch.cuda.synchronize()
    X0 = torch.from_numpy(st.maximal_to_minimal(Za.cpu().numpy())).cuda()
    # the law: x_ref = the state after the roll-in, seeded small gains (the same for every environment)
    K = torch.from_numpy(np.random.default_rng(7).normal(0.0, 0.05, (nu, 2 * nu))).cuda()
    # one (steps, envs) for every array of the law: x_ref is per environment, so K is given per environment as well (column-major)
    Kc = K.t().expand(B, 2 * nu, nu).contiguous()
    xr = X0.contiguous()
    Ua = torch.empty((T, B, nu), **f64)
    Zf, sts = torch.empty((B, nz), **f64), torch.empty(B, **i32)
    stream = torch.cuda.current_stream()
    s = stream.cuda_stream

    def fb():
        st.rollout_feedback_device(Za.data_ptr(), Zf.data_ptr(), B, T, Kc.data_ptr(), 1, B, dx_ref=xr.data_ptr(), dU_applied=Ua.data_ptr(),
                                   dstatus=sts.data_ptr(), opts=opts, stream=s)

    def roll():
        st.rollout_device(Za.data_ptr(), Ua.data_ptr(), Zf.data_ptr(), B, T, opts, dstatus=sts.data_ptr(), stream=s)

    def rollgen():
        gen.rollout_device(Za.data_ptr(), Ua.data_ptr(), Zf.data_ptr(), B, T, opts, dstatus=sts.data_ptr(), stream=s)

    Zp = [torch.empty((B, nz), **f64) for _ in range(2)]
    Xp, Up = torch.empty((B, 2 * nu), **f64), torch.empty((B, nu), **f64)

    def perstep():
        z = Za
        for t in range(T):
            st.maximal_to_minimal_device(z.data_ptr(), Xp.data_ptr(), B, stream=s)
            torch.mm(xr - Xp, K.t(), out=Up)  # u = -K (x - x_ref)
            st.step_device(z.data_ptr(), Up.data_ptr(), Zp[t % 2].data_ptr(), B, opts, stream=s)
            z = Zp[t % 2]

    arms = {"fb": fb, "roll": roll, "rollgen": rollgen, "perstep": perstep}
    fb()
    torch.cuda.synchronize()
    ref = Zf.clone()
    identical = True
    for k in ("roll", "rollgen"):
        Zf.zero_()
        arms[k]()
        torch.cuda.synchronize()
        identical &= bool(torch.equal(Zf, ref))
    for _ in range(warmup):
        for f in arms.values():
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    order = list(arms)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(repeats):
        for k in order[r % len(order):] + order[: r % len(order)]:
            ev0.record(stream)
            arms[k]()
            ev1.record(stream)
            ev1.synchronize()
            times[k].append(ev0.elapsed_time(ev1))
    res = {"mech": name, "B": B, "T": T, "repeats": repeats, "bit_identical": identical, "small_step": st.launch_config["small_step"]}
    for k in arms:
        med, iqr = _q(times[k])
        res[f"{k}_ms"], res[f"{k}_iqr_ms"] = round(med, 3), round(iqr, 3)
    for a, b in (("fb", "rollgen"), ("rollgen", "roll"), ("fb", "roll"), ("perstep", "fb")):
        res[f"{a}_over_{b}"] = round(_q(np.array(times[a]) / np.array(times[b]))[0], 4)
    res["fb_env_steps_per_s"] = round(B * T / (res["fb_ms"] * 1e-3))
    res["perstep_env_steps_per_s"] = round(B * T / (res["perstep_ms"] * 1e-3))
    st.close()
    gen.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mech", nargs="+", default=["ant"])
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    card = _card()
    out = []
    for name in a.mech:
        r = run(name, a.batch, a.steps, a.repeats, a.warmup)
        r["card"] = card
        print(f"{name} B={r['B']} T={r['T']} ({card}): fb {r['fb_ms']} ms (IQR {r['fb_iqr_ms']}), roll {r['roll_ms']} ms (IQR {r['roll_iqr_ms']}), "
              f"rollgen {r['rollgen_ms']} ms (IQR {r['rollgen_iqr_ms']}), perstep {r['perstep_ms']} ms (IQR {r['perstep_iqr_ms']}); "
              f"fb/rollgen {r['fb_over_rollgen']}, rollgen/roll {r['rollgen_over_roll']}, fb/roll {r['fb_over_roll']}, perstep/fb {r['perstep_over_fb']}; "
              f"bit-identical: {r['bit_identical']}", flush=True)
        out.append(r)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
