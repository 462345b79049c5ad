"""A/B timing of the forward step kernel specialised for small mechanisms against the generic one, on the states bench.py times.

    python tools/ab_step.py [--mech ant] [--batch 4096] [--pairs 40] [--warmup 5]
    python tools/ab_step.py --profile [--prof-lib LIB] [--mech ant] [--batch 4096]

Brings the bench.py workload of the mechanism to its timed state (same seeds, roll-in and episode restarts: bench's synthetic_batch,
random_inputs and WORKLOADS), then creates three steppers: two with DOJO_B200_GENERIC_STEP set (the generic kernel, "A" and its
repeat "A2") and one without ("B", the kernel dojo_create picks).  Every pair steps the same state with each of them in a rotating order, each
launch timed alone with CUDA events after a 256 MiB L2 flush, and checks that A and B return bit-identical next states, status and
iteration counts; the state then advances with A's result.  Prints per arm the median and interquartile range of the step time, the
median and IQR of the per-pair ratios A / B (speed-up of the specialised kernel) and A / A2 (the spread between repeats of one arm),
and one JSON line with the same numbers.

--profile runs tools/time_variant.py with DJ_PROF=1 on a DJ_PROFILE build of the library (built into a temporary directory unless
--prof-lib names one) for both arms, and prints its per-phase cycle breakdown per environment-step (eval_jac, eval_ls, fact, solve,
align, cone, center).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _stepper(mech, B, generic):
    from dojo_jl_b200.solver import BatchedStepper
    old = os.environ.pop("DOJO_B200_GENERIC_STEP", None)
    if generic:
        os.environ["DOJO_B200_GENERIC_STEP"] = "1"
    try:
        return BatchedStepper(mech, B)  # dojo_create reads the switch
    finally:
        os.environ.pop("DOJO_B200_GENERIC_STEP", None)
        if old is not None:
            os.environ["DOJO_B200_GENERIC_STEP"] = old


def _q(x):
    x = np.asarray(x, float)
    q1, med, q3 = np.percentile(x, [25, 50, 75])
    return float(med), float(q3 - q1)


def ab(name, B, pairs, warmup):
    import torch
    import bench
    import dojo_jl_b200 as dj
    from dojo_jl_b200 import capi
    mech = dj.get_mechanism(name)
    w = bench.WORKLOADS[name]
    opts = capi.solver_options()
    arms = {"A": _stepper(mech, B, True), "A2": _stepper(mech, B, True), "B": _stepper(mech, B, False)}
    small = {k: s.launch_config["small_step"] for k, s in arms.items()}
    Z0, rng = bench.synthetic_batch(mech, B, 0xD0D0 + 1, name)
    rollin, episode = w["rollin"], w["episode"]
    U = torch.from_numpy(bench.random_inputs(mech, rng, rollin + warmup + pairs, B, bench.SCALE.get(name, 1.0))).cuda()
    Z0d = torch.from_numpy(Z0).cuda()
    Za = Z0d.clone()
    out = {k: (torch.empty_like(Za), torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda")) for k in arms}
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream()

    def launch(k, t, Z):
        zn, st, it = out[k]
        arms[k].step_device(Z.data_ptr(), U[t].data_ptr(), zn.data_ptr(), B, opts, dstatus=st.data_ptr(), diters=it.data_ptr(), stream=stream.cuda_stream)

    for t in range(rollin):  # bench.py's untimed roll-in (forward only, no restarts)
        for k in arms:
            launch(k, t, Za)
        Za = out["A"][0].clone()
    k_global = 0
    times = {k: [] for k in arms}
    identical = True
    order = list(arms)
    for p in range(warmup + pairs):
        if episode and k_global % episode == 0:  # bench.py's episode restarts, counted over warm-up and timed steps
            Za.copy_(Z0d)
        t = rollin + p
        rot = order[p % 3:] + order[:p % 3]
        for k in rot:
            flush.fill_(p & 0xFF)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            launch(k, t, Za)
            e1.record(stream)
            torch.cuda.synchronize()
            if p >= warmup:
                times[k].append(e0.elapsed_time(e1))
        for k in ("A2", "B"):
            identical = identical and all(torch.equal(x, y) for x, y in zip(out["A"], out[k]))
        Za = out["A"][0].clone()
        k_global += 1
    ratio = np.asarray(times["A"]) / np.asarray(times["B"])
    rep = np.asarray(times["A"]) / np.asarray(times["A2"])
    rec = {"mechanism": name, "batch": B, "pairs": pairs, "small_step": small, "bit_identical": bool(identical),
           "gpu": torch.cuda.get_device_name(0)}
    for k in arms:
        rec[f"{k}_ms_median"], rec[f"{k}_ms_iqr"] = _q(times[k])
    rec["ratio_A_over_B_median"], rec["ratio_A_over_B_iqr"] = _q(ratio)
    rec["ratio_A_over_A2_median"], rec["ratio_A_over_A2_iqr"] = _q(rep)
    print(f"{name} B={B}, {pairs} pairs on {rec['gpu']}  (A, A2: DOJO_B200_GENERIC_STEP; B: default; small_step {small})")
    for k in arms:
        print(f"  {k:2s}: median {rec[f'{k}_ms_median']:8.3f} ms  IQR {rec[f'{k}_ms_iqr']:.3f} ms  ({B / rec[f'{k}_ms_median'] * 1e3:,.0f} env-steps/s)")
    print(f"  A / B  per pair: median {rec['ratio_A_over_B_median']:.4f}  IQR {rec['ratio_A_over_B_iqr']:.4f}")
    print(f"  A / A2 per pair: median {rec['ratio_A_over_A2_median']:.4f}  IQR {rec['ratio_A_over_A2_iqr']:.4f}  (repeats of one arm)")
    print(f"  outputs (states, status, iterations) bit-identical: {identical}")
    print(json.dumps(rec))
    return rec


def profile(name, B, lib, steps):
    if lib is None:
        sys.path.insert(0, os.path.join(ROOT, "dojo.jl_b200"))
        import build
        lib = build.build(force=True, defines=["DJ_PROFILE"], out=os.path.join(tempfile.mkdtemp(prefix="dojo_prof_"), "libdojo_b200_prof.so"))
    for arm, generic in (("A (generic)", True), ("B (default)", False)):
        env = dict(os.environ, DJ_PROF="1", DJ_ROLLOUT="0")
        env.pop("DOJO_B200_GENERIC_STEP", None)
        if generic:
            env["DOJO_B200_GENERIC_STEP"] = "1"
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "time_variant.py"), lib, name, str(B), str(steps)], env=env, capture_output=True,
                           text=True, cwd=ROOT)
        print(f"--- {arm}")
        print(r.stdout.rstrip())
        if r.returncode != 0:
            print(r.stderr[-3000:])
            raise SystemExit(r.returncode)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--mech", default="ant")
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--pairs", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="per-phase cycle breakdown of both arms (DJ_PROFILE build)")
    ap.add_argument("--prof-lib", default=None, help="a DJ_PROFILE build of libdojo_b200.so (default: build one in a temporary directory)")
    ap.add_argument("--prof-steps", type=int, default=20)
    a = ap.parse_args()
    if a.pairs < 40:
        ap.error("--pairs: at least 40 pairs")
    if a.profile:
        profile(a.mech, a.batch, a.prof_lib, a.prof_steps)
    else:
        ab(a.mech, a.batch, a.pairs, a.warmup)


if __name__ == "__main__":
    main()
