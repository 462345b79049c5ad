"""Cost of the traced step: dojo_step_trace_async against dojo_step_async on the benchmarked ant batch, timed with CUDA events.

    python tools/trace_cost.py [--B 4096] [--reps 40] [--out DIR]

The batch is bench.py's ant workload (seeded states after its roll-in).  Both variants step the same input states again and again and
are alternated call by call, so that clock and co-tenant drift hit both alike; each call is timed on its own by a pair of events.
Prints one JSON line: the GPU's name and power limit, the median and quartiles per variant and the median ratio.  Also checks that
both variants computed the same next states, status and iteration counts.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import bench  # noqa: E402
import dojo_jl_b200 as dj  # noqa: E402
from dojo_jl_b200 import capi  # noqa: E402
from dojo_jl_b200.solver import BatchedStepper  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
        return name, power
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("trace_cost.py needs a CUDA device")
    mech, B = dj.get_mechanism("ant"), args.B
    opts = capi.solver_options()
    w = bench.WORKLOADS["ant"]
    Z, rng = bench.synthetic_batch(mech, B, 0xD0D0 + 1, "ant")
    U = bench.random_inputs(mech, rng, w["rollin"] + 1, B, bench.SCALE["ant"])
    st = BatchedStepper(mech, B)
    for t in range(w["rollin"]):
        Z = st.step(Z, U[t])[0]
    dev = torch.device("cuda:0")
    zin = torch.from_numpy(np.ascontiguousarray(Z)).to(dev)
    u = torch.from_numpy(np.ascontiguousarray(U[w["rollin"]])).to(dev)
    zout = {v: torch.empty_like(zin) for v in ("plain", "traced")}
    status = {v: torch.empty(B, dtype=torch.int32, device=dev) for v in zout}
    iters = {v: torch.empty(B, dtype=torch.int32, device=dev) for v in zout}
    trace = torch.empty((B, opts.max_iter, 5), dtype=torch.float64, device=dev)
    stream = torch.cuda.current_stream()

    def launch(v):
        st.step_device(zin.data_ptr(), u.data_ptr(), zout[v].data_ptr(), B, opts, dstatus=status[v].data_ptr(), diters=iters[v].data_ptr(),
                       stream=stream.cuda_stream, dtrace=trace.data_ptr() if v == "traced" else None)

    for _ in range(5):  # warm-up: module loading, the traced kernel's first use, the work-queue order of this batch
        launch("plain")
        launch("traced")
    torch.cuda.synchronize()
    times = {"plain": [], "traced": []}
    for k in range(args.reps):
        for v in (("plain", "traced") if k % 2 == 0 else ("traced", "plain")):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            launch(v)
            b.record(stream)
            b.synchronize()
            times[v].append(a.elapsed_time(b))
    same = all(torch.equal(x["plain"], x["traced"]) for x in (zout, status, iters))
    name, power = gpu_info()
    q = {v: np.percentile(times[v], [25, 50, 75]).tolist() for v in times}
    ratio = float(np.median(np.array(times["traced"]) / np.array(times["plain"])))
    rec = {"gpu": name, "power_limit": power, "mech": "ant", "B": B, "reps": args.reps, "ms_plain_q25_q50_q75": q["plain"],
           "ms_traced_q25_q50_q75": q["traced"], "median_ratio_traced_over_plain": ratio, "outputs_identical": same,
           "mean_iters": float(iters["plain"].float().mean())}
    print(json.dumps(rec))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "trace_cost.json"), "w") as f:
            f.write(json.dumps(rec) + "\n")
    if not same:
        raise SystemExit("traced and untraced steps differ")


if __name__ == "__main__":
    main()
