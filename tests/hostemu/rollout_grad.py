"""The trajectory Jacobians of a fused rollout on the CPU -- TEST INFRASTRUCTURE for tests/test_rollout_grad.py.

RolloutGradEmu reaches one more entry point of the kernel emulation (driver.inc): hostemu_rollout_grad runs the recording rollout
dojo_step_kernel<false, false, false, false, REC = true> on CPU fibers, publishing every (environment, step) pair t * B + e, and then
the gradient kernel over the B * T pairs in the order they were published, as dojo_rollout_grad does."""
import ctypes as C

import numpy as np

from dojo_jl_b200 import capi
from .harness import HostEmu, _p


class RolloutGradEmu(HostEmu):
    """HostEmu's kernels (step, step_grad, kinjac) and the recording rollout with its gradients (rollout_grad)."""

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
