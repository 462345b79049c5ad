"""Write tests/golden/ldu_emulation.npz: steps and gradients of the kernel emulation (tests/hostemu) on fixed inputs.

    python tools/make_ldu_golden.py [out.npz]

tests/test_ldu_program.py replays the same inputs on the emulation of the current sources and requires every array to be
bit-identical.  The file was written from the revision before the block LDU read its steps from the plan's LDU program (dojo_plan.h
LduOp), so it pins that the program changes no floating-point operation: states, status, Newton iterations, full solution vectors
and the state / input Jacobians (by digest), at 1 and 4 environments per CTA.  Inputs come from fixed seeds; nothing else is read.
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

OUT = os.path.join(ROOT, "tests", "golden", "ldu_emulation.npz")
# (key, mechanism, get_mechanism overrides): the BASELINE models, a joint-limited hopper and a block on LinearContact
CASES = (("pendulum", "pendulum", {}), ("ant", "ant", {}), ("quadruped", "quadruped", {}), ("atlas", "atlas", {}),
         ("raiberthopper", "raiberthopper", {}), ("block_linear", "block", {"contact_type": "linear"}))
SLOTS = (1, 4)
B = 4


def inputs(mech, seed):
    from conftest import jittered_states, random_inputs
    rng = np.random.default_rng(seed)
    Z = jittered_states(mech, B, rng)
    U = random_inputs(mech, B, rng, 0.5)
    return Z, U


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def run(key, name, over, seed):
    """every array the test compares, keyed '<case>/<slots>/<what>'"""
    import dojo_jl_b200 as dj
    from hostemu.harness import HostEmu
    mech = dj.get_mechanism(name, **over)
    emu = HostEmu(mech)
    Z, U = inputs(mech, seed)
    out = {}
    for slots in SLOTS:
        Zn, st, it, sol = emu.step(Z, U, slots=slots)
        p = f"{key}/{slots}/"
        out.update({p + "Zn": Zn, p + "status": st, p + "iters": it, p + "sol": sol})
        g = emu.step_grad(Z, U, slots=slots, slots_grad=slots)
        # the Jacobians by SHA-256 of their bytes (atlas: 372 x 372 per environment would make the file megabytes)
        out.update({p + "gZn": g[0], p + "Fz_sha256": digest(g[1]), p + "Fu_sha256": digest(g[2]), p + "gstatus": g[3], p + "giters": g[4]})
    return out


def generate():
    out = {}
    for seed, (key, name, over) in enumerate(CASES):
        out.update(run(key, name, over, 100 + seed))
    return out


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else OUT
    arrays = generate()
    np.savez_compressed(path, **arrays)
    print(f"wrote {len(arrays)} arrays to {path}")
