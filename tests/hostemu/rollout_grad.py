"""The trajectory Jacobians of a fused rollout on the CPU -- TEST INFRASTRUCTURE for tests/test_rollout_grad.py.

RolloutGradEmu builds the kernel emulation TU of gen.py (generated from the unmodified sources, like tests/hostemu/trace.py and
small.py) with one more entry point: hostemu_rollout_grad runs the recording rollout dojo_step_kernel<false, false, false, false,
REC = true> on CPU fibers, publishing every (environment, step) pair t * B + e, and then the gradient kernel over the B * T pairs in the
order they were published, as dojo_rollout_grad does.  The other entry points of driver.inc stay as they are.  The library is built
into tests/hostemu/_build (or a temporary directory when the tree is read-only)."""
import ctypes as C
import os

import numpy as np

from dojo_jl_b200 import capi
from . import gen
from .harness import HostEmu, _ip, _p, _vp
from .trace import _build_dir, _compile, _stale, _substitute

_EMU_ENTRY = r"""
// dojo_rollout_grad on the emulation: traj [nz x B x (T + 1)] holds Z0 in slab 0; Fz / Fu / status / iters per pair t * B + e
extern "C" int hostemu_rollout_grad(void* p, const DojoSolverOptions* opts, int B, int T, double* traj, const double* U, double* Fz, double* Fu,
                                    int32_t* status, int32_t* iters, int slots, int slots_grad, int smem_plan, int grid) {
  DojoHandle* h = static_cast<EmuHandle*>(p)->h;
  if (!h->grad_bytes) return -1;
  const int pairs = B * T;
  std::vector<double> sol_raw((size_t)pairs * h->plan.nres);
  std::vector<int> done(pairs + 2, -1);
  done[0] = 0; done[1] = 0;
  int counter = 0;
  StepArgs a = emu_args(h, opts, B, false, slots, smem_plan != 0, &counter);
  a.Z = traj; a.U = U; a.traj = traj + (size_t)B * h->plan.nz; a.T = T; a.sol_raw = sol_raw.data(); a.status = status; a.iters = iters;
  a.done_count = done.data(); a.done_list = done.data() + 2;
  const size_t smem = slots * h->arena_bytes + (smem_plan ? h->blob_bytes : 0);
  for (int b = 0; b < grid; ++b) emu::run_cta(b, grid, 32 * h->nw * slots, smem, [&a] { dojo_step_kernel<false, false, false, false, true>(a); });
  int counter2 = 0;
  StepArgs g = emu_args(h, opts, pairs, true, slots_grad, smem_plan != 0, &counter2);
  g.Z = traj; g.U = U; g.sol_raw = sol_raw.data(); g.status = status; g.Fz = Fz; g.Fu = Fu;
  g.done_list = done.data() + 2;
  emu_launch<true>(h, g, 1, slots_grad, smem_plan != 0);
  return 0;
}
"""


def build_emulation() -> str:
    name = "libdojo_hostemu_rollout_grad_fma.so" if gen.FMA else "libdojo_hostemu_rollout_grad.so"
    lib = os.path.join(_build_dir(), name)
    if not _stale(lib, gen.DEPS + [os.path.abspath(__file__)]):
        return lib
    here = gen.HERE
    text = open(gen.generate()).read()
    text = _substitute(text, [('#include "../cuda_shim.h"', f'#include "{os.path.join(here, "cuda_shim.h")}"'),
                              ('#include "../driver.inc"', f'#include "{os.path.join(here, "driver.inc")}"')], "the emulation TU")
    fp = ["-ffp-contract=fast", "-march=x86-64-v3"] if gen.FMA else ["-ffp-contract=off"]
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared"] + fp + ["-Wno-unknown-pragmas", "-Wno-unused-function", "-Wno-unused-variable",
                                                                         "-Wno-unused-but-set-variable"]
    return _compile(text + _EMU_ENTRY, name, cmd)


class RolloutGradEmu(HostEmu):
    """HostEmu's kernels (step, step_grad, kinjac) and the recording rollout with its gradients (rollout_grad) in one library."""

    def __init__(self, mech):
        L = C.CDLL(build_emulation())
        op = C.POINTER(capi.DojoSolverOptions)
        L.hostemu_rollout_grad.argtypes = [_vp, op, _ip, _ip, _vp, _vp, _vp, _vp, _vp, _vp, _ip, _ip, _ip, _ip]
        L.hostemu_rollout_grad.restype = C.c_int
        L.hostemu_create.restype = _vp
        L.hostemu_create.argtypes = [C.POINTER(capi.DojoMechanismDesc)]
        L.hostemu_destroy.argtypes = [_vp]
        L.hostemu_last_error.restype = C.c_char_p
        for n in ("hostemu_num_residual", "hostemu_num_input", "hostemu_warps_per_env"):
            getattr(L, n).argtypes = [_vp]
        L.hostemu_step.argtypes = [_vp, op, _ip, _ip, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint32, _ip, _ip, _ip, _vp]
        L.hostemu_step_grad.argtypes = [_vp, op, _ip, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ip, _ip, _ip, _ip, _vp]
        L.hostemu_kinjac.argtypes = [_vp, _ip, _ip, _ip, _vp, _vp, _vp, _vp, _vp, _vp]
        self.L, self.mech = L, mech
        desc, self._keep = capi.flatten(mech)
        h = L.hostemu_create(C.byref(desc))
        if not h:
            raise RuntimeError("hostemu_create failed: " + L.hostemu_last_error().decode())
        self.h = C.c_void_p(h)
        assert L.hostemu_num_residual(self.h) == mech.nres and L.hostemu_num_input(self.h) == mech.nu

    def rollout_grad(self, Z0, U=None, T=1, opts=None, slots=1, slots_grad=1, smem_plan=True, grid=1):
        """dojo_rollout_grad, U [T, B, nu].  Returns (Z_traj [T+1, B, nz], Fz [T, B, 12Nb, 12Nb], Fu [T, B, 12Nb, nu], status [T, B],
        iters [T, B])."""
        Z0 = np.ascontiguousarray(np.atleast_2d(Z0), dtype=np.float64)
        B, ng, nu = Z0.shape[0], 12 * self.mech.Nb, self.mech.nu
        U = np.zeros((T, B, nu)) if U is None else np.ascontiguousarray(U, dtype=np.float64)
        assert U.shape == (T, B, nu)
        traj = np.empty((T + 1, B, Z0.shape[1]))
        traj[0] = Z0
        Fz, Fu = np.empty((T, B, ng, ng)), np.empty((T, B, nu, ng))
        st, it = np.zeros((T, B), dtype=np.int32), np.zeros((T, B), dtype=np.int32)
        o = opts if opts is not None else capi.solver_options()
        rc = self.L.hostemu_rollout_grad(self.h, C.byref(o), B, T, _p(traj), _p(U), _p(Fz), _p(Fu), _p(st), _p(it), slots, slots_grad, int(smem_plan), grid)
        if rc != 0:
            raise RuntimeError("the gradient workspace does not fit for this mechanism")
        return traj, Fz.transpose(0, 1, 3, 2), Fu.transpose(0, 1, 3, 2), st, it


def rollout_minimal_gradients(em, hc, X0, U, T, opts=None, slots=2, slots_grad=2):
    """dojo_rollout_minimal_gradients as the library composes it, on the emulation (em: RolloutGradEmu) and the host build of the map
    kernels (hc: hostcheck.harness.HostCheck): the maximal rollout from minimal_to_maximal(X0), the map-Jacobian kernel between slabs t
    and t + 1, maximal_to_minimal of every slab.  Returns (X_traj [T+1, B, 2nu], Gx [T, B, 2nu, 2nu], Gu [T, B, 2nu, nu], status, iters)."""
    traj, Fz, Fu, st, it = em.rollout_grad(hc.minimal_to_maximal(np.atleast_2d(X0)), U, T, opts, slots=slots, slots_grad=slots_grad)
    B = traj.shape[1]
    Gx, Gu = hc.minimal_gradients(traj[:-1].reshape(T * B, -1), traj[1:].reshape(T * B, -1), Fz.reshape(T * B, *Fz.shape[2:]),
                                  Fu.reshape(T * B, *Fu.shape[2:]))
    X = hc.maximal_to_minimal(traj.reshape((T + 1) * B, -1)).reshape(T + 1, B, -1)
    return X, Gx.reshape(T, B, *Gx.shape[1:]), Gu.reshape(T, B, *Gu.shape[1:]), st, it
