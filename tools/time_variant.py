"""Time one build variant: python tools/time_variant.py <lib.so> mech B steps  (DOJO_B200_LIB overrides the library path)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import dojo_jl_b200 as dj
from dojo_jl_b200 import solver
solver.LIB_PATH = os.path.abspath(sys.argv[1])
from dojo_jl_b200.solver import BatchedStepper
import bench
name, B, steps = sys.argv[2], int(sys.argv[3]), int(sys.argv[4])
mech = dj.get_mechanism(name)
Z0, rng = bench.synthetic_batch(mech, B, 0xD0D0 + 1)
U = torch.from_numpy(bench.random_inputs(mech, rng, 20 + steps, B, bench.SCALE[name])).cuda()
s = BatchedStepper(mech, B)
Za = torch.from_numpy(Z0).cuda(); Zb = torch.empty_like(Za)
it = torch.zeros(B, dtype=torch.int32, device="cuda")
st = torch.cuda.current_stream().cuda_stream
for t in range(20):
    s.step_device(Za.data_ptr(), U[t].data_ptr(), Zb.data_ptr(), B, stream=st); Za, Zb = Zb, Za
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
its = 0
for t in range(20, 20 + steps):
    s.step_device(Za.data_ptr(), U[t].data_ptr(), Zb.data_ptr(), B, diters=it.data_ptr(), stream=st); Za, Zb = Zb, Za
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / steps
print(f"{os.path.basename(sys.argv[1]):20s} {name} B={B}: {ms:8.3f} ms/step  {B/ms*1e3:10.0f} env-steps/s  smem/env {s.shared_bytes_per_env}  checksum {float(Za.sum()):.9f}")
if hasattr(s, "rollout_device") and os.environ.get("DJ_ROLLOUT", "1") != "0":
    # fused rollout: the same `steps` steps in ONE launch (environment-resident across steps)
    Zr = Za.clone(); Zf = torch.empty_like(Za)
    Ur = U[20:20 + steps].contiguous()
    s.rollout_device(Zr.data_ptr(), Ur.data_ptr(), Zf.data_ptr(), B, steps, stream=st)
    torch.cuda.synchronize()
    e0.record()
    s.rollout_device(Zr.data_ptr(), Ur.data_ptr(), Zf.data_ptr(), B, steps, stream=st)
    e1.record(); torch.cuda.synchronize()
    msr = e0.elapsed_time(e1) / steps
    print(f"{'':20s} fused rollout T={steps}: {msr:8.3f} ms/step  {B/msr*1e3:10.0f} env-steps/s")
if os.environ.get("DJ_PROF"):
    import ctypes as C
    out = (C.c_ulonglong * 32)()
    s.L.dojo_debug_cycles.argtypes = [C.c_void_p, C.c_void_p]
    s.L.dojo_debug_cycles(s.h, out)
    tot = sum(out)
    names = ("eval_jac", "eval_ls", "fact", "solve", "misc", "f_fold", "f_inv", "f_rm", "f_schur", "f_bar", "-", "-", "-", "-", "align", "cone", "center",
             "rolewait_w0", "rolewait_w1", "-", "-", "-", "-", "-", "-", "s_cond", "s_fwd", "s_bwd", "s_rec", "s_bar")
    print("   cycles/env-step: " + "  ".join(f"{n}={v/ (B*(20+steps)):.0f}" for n, v in zip(names, out) if n != "-"))
