"""Timing of the trajectory Jacobians: dojo_rollout_grad_async against the two ways of getting them from single-step gradients.

    python tools/rollout_grad_time.py [--mech ant quadruped] [--batch 1024] [--steps 32] [--repeats 15] [--warmup 2]

Per mechanism, from bench.py's seeded batch after its roll-in (synthetic_batch, random_inputs, WORKLOADS) and T seeded inputs:
  seq    T x dojo_step_grad_async, each from the state the previous one returned (two launches per step, each waiting for its slowest
         environment);
  flat   one dojo_step_grad_async over the B * T (state, input) pairs of a recorded dojo_rollout (every step solved a second time;
         needs B * T <= max_batch);
  fused  one dojo_rollout_grad_async (the recording rollout, with the gradient kernel consuming its pairs as they finish);
  roll   the dojo_rollout_async that records the states flat reads (flat's full cost is roll + flat).
seq, flat and fused write the same device buffers; each repeat runs the arms in a rotating order, each call timed alone with CUDA
events.  Before timing, the Jacobians, states, status and iterations of the three are checked to be bit-identical.  Prints the median
and interquartile range per arm, the medians of the per-repeat ratios seq / fused, flat / fused and (flat + roll) / fused, the card and
its power limit, and one JSON line.
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
    st = BatchedStepper(mech, B * T)
    nz, nu, ng = st.nz, st.nu, st.ngrad
    Z0, rng = bench.synthetic_batch(mech, B, 0xD0D0 + 1, name)
    U = torch.from_numpy(bench.random_inputs(mech, rng, w["rollin"] + T, B, bench.SCALE.get(name, 1.0))).cuda()
    Za, Zb = torch.from_numpy(Z0).cuda(), torch.empty((B, nz), dtype=torch.float64, device="cuda")
    for t in range(w["rollin"]):
        st.step_device(Za.data_ptr(), U[t].data_ptr(), Zb.data_ptr(), B, opts)
        Za, Zb = Zb, Za
    U = U[w["rollin"]:].contiguous()
    f64, i32 = dict(dtype=torch.float64, device="cuda"), dict(dtype=torch.int32, device="cuda")
    traj = torch.empty((T + 1, B, nz), **f64)
    traj[0] = Za
    Zscratch = torch.empty((T * B, nz), **f64)
    Fz, Fu = torch.empty((T, B, ng, ng), **f64), torch.empty((T, B, nu, ng), **f64)
    sts, its = torch.empty((T, B), **i32), torch.empty((T, B), **i32)
    stream = torch.cuda.current_stream()
    s = stream.cuda_stream

    def seq():
        for t in range(T):
            st.step_grad_device(traj[t].data_ptr(), U[t].data_ptr(), traj[t + 1].data_ptr(), Fz[t].data_ptr(), Fu[t].data_ptr(), B, opts,
                                dstatus=sts[t].data_ptr(), diters=its[t].data_ptr(), stream=s)

    # the flattened arm reads the states of a recorded rollout: slabs 0 .. T - 1 of the trajectory (recorded once, untimed)
    rec = torch.empty((T + 1, B, nz), **f64)
    rec[0] = Za
    Zf = torch.empty((B, nz), **f64)
    st.rollout_device(rec[0].data_ptr(), U.data_ptr(), Zf.data_ptr(), B, T, opts, dtraj=rec[1].data_ptr(), stream=s)

    def flat():
        st.step_grad_device(rec.data_ptr(), U.data_ptr(), Zscratch.data_ptr(), Fz.data_ptr(), Fu.data_ptr(), B * T, opts, dstatus=sts.data_ptr(),
                            diters=its.data_ptr(), stream=s)

    def roll():
        st.rollout_device(rec[0].data_ptr(), U.data_ptr(), Zf.data_ptr(), B, T, opts, dtraj=rec[1].data_ptr(), stream=s)

    def fused():
        st.rollout_grad_device(traj.data_ptr(), U.data_ptr(), traj.data_ptr(), Fz.data_ptr(), Fu.data_ptr(), B, T, opts, dstatus=sts.data_ptr(),
                               diters=its.data_ptr(), stream=s)

    arms = {"seq": seq, "flat": flat, "fused": fused, "roll": roll}
    # identical results: fused is the reference; flat writes its next states to scratch, so its trajectory is compared with the record
    fused()
    torch.cuda.synchronize()
    ref = [x.clone() for x in (traj, Fz, Fu, sts, its)]
    identical = bool(torch.equal(rec, ref[0]))
    for k in ("seq", "flat"):
        Fz.zero_(); Fu.zero_(); sts.fill_(-1); its.fill_(-1)
        if k == "seq":
            traj[1:].zero_()
        arms[k]()
        torch.cuda.synchronize()
        identical &= all(torch.equal(a, b) for a, b in zip((traj, Fz, Fu, sts, its), ref))
    del ref
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
    res = {"mech": name, "B": B, "T": T, "repeats": repeats, "bit_identical": identical}
    for k in arms:
        med, iqr = _q(times[k])
        res[f"{k}_ms"], res[f"{k}_iqr_ms"] = round(med, 3), round(iqr, 3)
    res["flat_plus_roll_over_fused"] = round(_q((np.array(times["flat"]) + np.array(times["roll"])) / np.array(times["fused"]))[0], 3)
    for k in ("seq", "flat"):
        res[f"{k}_over_fused"] = round(_q(np.array(times[k]) / np.array(times["fused"]))[0], 3)
    st.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mech", nargs="+", default=["ant", "quadruped"])
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    card = _card()
    out = []
    for name in a.mech:
        r = run(name, a.batch, a.steps, a.repeats, a.warmup)
        r["card"] = card
        print(f"{name} B={r['B']} T={r['T']} ({card}): seq {r['seq_ms']} ms (IQR {r['seq_iqr_ms']}), flat {r['flat_ms']} ms (IQR {r['flat_iqr_ms']}), "
              f"fused {r['fused_ms']} ms (IQR {r['fused_iqr_ms']}), roll {r['roll_ms']} ms; seq/fused {r['seq_over_fused']}, flat/fused {r['flat_over_fused']}, "
              f"(flat + roll)/fused {r['flat_plus_roll_over_fused']}; "
              f"bit-identical: {r['bit_identical']}", flush=True)
        out.append(r)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
