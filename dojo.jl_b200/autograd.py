"""PyTorch autograd through a fused rollout: rollout(mechanism, Z0, U) is differentiable with respect to Z0 and U, and
rollout_feedback(mechanism, Z0, K, ...) through a closed loop with respect to Z0 and the linear law's tensors.  The coordinate maps
minimal_to_maximal / maximal_to_minimal are differentiable too, so rollout_minimal(mechanism, X0, U) starts from and returns minimal
states, and rollout_feedback(mechanism, minimal_to_maximal(mechanism, X0), K, ...) backpropagates to a minimal start.

    from dojo_jl_b200.autograd import rollout
    Z_traj, status = rollout(mech, Z0, U)           # CUDA fp64: Z0 [B, 13Nb], U [T, B, nu] -> Z_traj [T+1, B, 13Nb], status [T, B]
    loss = f(Z_traj); loss.backward()               # Z0.grad, U.grad

The forward pass records the rollout on the device (dojo_rollout_tape: the trajectory and the final solver iterate of every step) on the
current torch stream; the backward pass runs one adjoint pass over it (dojo_rollout_vjp), also on the current stream.  Nothing of size
12Nb x 12Nb per step is formed.  The gradients are those of the implicit-function-theorem Jacobians dojo_rollout_grad returns.

Quaternions.  A state holds each body's attitude as a unit quaternion q, and the library differentiates along attitude perturbations
q (x) (1, d) (dz in [x, v, phi, w] per body, 12 entries).  With G(q) = d(q (x) (1, d)) / dd at d = 0 (4 x 3; the reference's LVᵀmat(q)):
  * a cotangent qbar on a quaternion of Z_traj enters the adjoint pass as phibar = G(q)' qbar;
  * the quaternion part of dL/dZ0 is returned as G(q0) phibar0, the gradient in the tangent space of the unit sphere at q0: its radial
    component q0' (dL/dq0) is 0.  A loss that depends on |q0| (it should not: Z0's quaternions are unit) is not differentiated along it.
to_attitude / from_attitude are these two maps; they take torch tensors or numpy arrays alike (the CPU tests use the numpy form).
status [T, B] (not differentiable) is each step's solver status; an environment whose backward pass meets a non-finite factorisation gets
NaN gradients.
"""
import numpy as np

from .mechanism import Mechanism
from .solver import BatchedStepper


def _xp(a):
    return np if isinstance(a, np.ndarray) else __import__("torch")


def attitude_map(q):
    """G(q) [..., 4, 3] = d(q (x) (1, d)) / dd for quaternions q [..., 4] = (s, x, y, z):  [-v'; s I + skew(v)]"""
    xp = _xp(q)
    s, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    rows = [(-x, -y, -z), (s, -z, y), (z, s, -x), (-y, x, s)]
    return xp.stack([xp.stack(r, -1) for r in rows], -2)


def to_attitude(Z, gZ):
    """cotangents in the state packing [x, v, q, w] per body (gZ [..., 13Nb], at the states Z [..., 13Nb]) -> the gradients' packing
    [x, v, phi, w] (12Nb), phibar = G(q)' qbar"""
    xp = _xp(gZ)
    sh = gZ.shape[:-1]
    g = gZ.reshape(sh + (-1, 13))
    q = Z.reshape(sh + (-1, 13))[..., 6:10]
    phi = xp.einsum("...ij,...i->...j", attitude_map(q), g[..., 6:10])
    return xp.concatenate([g[..., :6], phi, g[..., 10:]], -1).reshape(sh + (-1,))


def from_attitude(Z, g):
    """the gradients' packing [x, v, phi, w] per body (g [..., 12Nb], at the states Z [..., 13Nb]) -> the state packing, qbar = G(q) phibar
    (tangent to the unit sphere at q)"""
    xp = _xp(g)
    sh = g.shape[:-1]
    g = g.reshape(sh + (-1, 12))
    q = Z.reshape(sh + (-1, 13))[..., 6:10]
    qb = xp.einsum("...ij,...j->...i", attitude_map(q), g[..., 6:9])
    return xp.concatenate([g[..., :6], qb, g[..., 9:]], -1).reshape(sh + (-1,))


_steppers = {}


def _stepper(mech: Mechanism, B: int, device: int) -> BatchedStepper:
    """one handle per (mechanism, device), replaced by a larger one when B outgrows it; a replaced handle stays alive while a recorded
    rollout holds it for its backward pass"""
    key = (id(mech), device)
    s = _steppers.get(key)
    if s is None or s.max_batch < B:
        s = BatchedStepper(mech, max(B, 64), device)
        _steppers[key] = s
    return s


def _function():
    import torch

    class Rollout(torch.autograd.Function):
        @staticmethod
        def forward(ctx, Z0, U, stepper, opts):
            T, B = U.shape[0], U.shape[1]
            dev = Z0.device
            Z0c, Uc = Z0.detach().contiguous(), U.detach().contiguous()
            Z_traj = torch.empty((T + 1, B, stepper.nz), dtype=torch.float64, device=dev)
            tape = torch.empty((T, B, stepper.nres), dtype=torch.float64, device=dev)
            status = torch.empty((T, B), dtype=torch.int32, device=dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
            stepper.rollout_tape_device(Z0c.data_ptr(), Uc.data_ptr() if stepper.nu > 0 else None, Z_traj.data_ptr(), tape.data_ptr(), B, T, opts,
                                        dstatus=status.data_ptr(), stream=stream)
            ctx.save_for_backward(Z_traj, Uc, tape)
            ctx.stepper = stepper
            ctx.mark_non_differentiable(status)
            return Z_traj, status

        @staticmethod
        def backward(ctx, gZ_traj, _gstatus):
            Z_traj, U, tape = ctx.saved_tensors
            s = ctx.stepper
            T, B = tape.shape[0], tape.shape[1]
            dev = Z_traj.device
            if gZ_traj is None:
                gZ_traj = torch.zeros_like(Z_traj)
            g = to_attitude(Z_traj, gZ_traj.to(torch.float64)).contiguous()
            gZ0 = torch.empty((B, s.ngrad), dtype=torch.float64, device=dev)
            gU = torch.empty((T, B, s.nu), dtype=torch.float64, device=dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
            s.rollout_vjp_device(Z_traj.data_ptr(), U.data_ptr() if s.nu > 0 else None, tape.data_ptr(), g.data_ptr(), gZ0.data_ptr(), B, T,
                                 dgU=gU.data_ptr() if s.nu > 0 else None, stream=stream)
            return from_attitude(Z_traj[0], gZ0), gU, None, None

    return Rollout


_Rollout = None


def rollout(mechanism: Mechanism, Z0, U, opts=None):
    """T open-loop steps of B environments, differentiable with respect to Z0 [B, 13Nb] and U [T, B, nu] (CUDA float64 tensors on one
    device).  Returns (Z_traj [T+1, B, 13Nb] with Z_traj[0] = Z0, status [T, B] int32).  opts: capi.solver_options(...) or None."""
    import torch
    global _Rollout
    if _Rollout is None:
        _Rollout = _function()
    if Z0.dtype != torch.float64 or U.dtype != torch.float64 or not Z0.is_cuda or U.device != Z0.device:
        raise ValueError("rollout: Z0 and U must be float64 CUDA tensors on one device")
    if Z0.dim() != 2 or U.dim() != 3 or U.shape[1] != Z0.shape[0] or Z0.shape[1] != mechanism.nz or U.shape[2] != mechanism.nu:
        raise ValueError(f"rollout: Z0 [B, {mechanism.nz}] and U [T, B, {mechanism.nu}] expected, got {tuple(Z0.shape)} and {tuple(U.shape)}")
    s = _stepper(mechanism, Z0.shape[0], Z0.device.index if Z0.device.index is not None else torch.cuda.current_device())
    return _Rollout.apply(Z0, U, s, opts)


def _map_functions():
    import torch
    from torch.autograd.function import once_differentiable

    def flat(a, k):  # [..., k] -> contiguous [n, k]
        return a.detach().reshape(-1, k).contiguous()

    class MinimalToMaximal(torch.autograd.Function):
        @staticmethod
        def forward(ctx, X, stepper):
            Xc = flat(X, stepper.nmin)
            n = Xc.shape[0]
            Z = torch.empty((n, stepper.nz), dtype=torch.float64, device=X.device)
            stepper.minimal_to_maximal_device(Xc.data_ptr(), Z.data_ptr(), n, stream=torch.cuda.current_stream(X.device).cuda_stream)
            ctx.save_for_backward(Z)
            ctx.stepper, ctx.shape = stepper, X.shape
            return Z.reshape(X.shape[:-1] + (stepper.nz,))

        @staticmethod
        @once_differentiable
        def backward(ctx, gZ):
            (Z,) = ctx.saved_tensors
            s = ctx.stepper
            g = to_attitude(Z, gZ.to(torch.float64).reshape(Z.shape)).contiguous()
            gX = torch.empty((Z.shape[0], s.nmin), dtype=torch.float64, device=Z.device)
            s.minimal_to_maximal_vjp_device(Z.data_ptr(), g.data_ptr(), gX.data_ptr(), Z.shape[0], stream=torch.cuda.current_stream(Z.device).cuda_stream)
            return gX.reshape(ctx.shape), None

    class MaximalToMinimal(torch.autograd.Function):
        @staticmethod
        def forward(ctx, Z, stepper):
            Zc = flat(Z, stepper.nz)
            n = Zc.shape[0]
            X = torch.empty((n, stepper.nmin), dtype=torch.float64, device=Z.device)
            stepper.maximal_to_minimal_device(Zc.data_ptr(), X.data_ptr(), n, stream=torch.cuda.current_stream(Z.device).cuda_stream)
            ctx.save_for_backward(Zc)
            ctx.stepper, ctx.shape = stepper, Z.shape
            return X.reshape(Z.shape[:-1] + (stepper.nmin,))

        @staticmethod
        @once_differentiable
        def backward(ctx, gX):
            (Z,) = ctx.saved_tensors
            s = ctx.stepper
            g = gX.to(torch.float64).reshape(Z.shape[0], s.nmin).contiguous()
            gZ = torch.empty((Z.shape[0], s.ngrad), dtype=torch.float64, device=Z.device)
            s.maximal_to_minimal_vjp_device(Z.data_ptr(), g.data_ptr(), gZ.data_ptr(), Z.shape[0], stream=torch.cuda.current_stream(Z.device).cuda_stream)
            return from_attitude(Z, gZ).reshape(ctx.shape), None

    return MinimalToMaximal, MaximalToMinimal


_MinimalToMaximal = _MaximalToMinimal = None


def _map_inputs(mechanism: Mechanism, a, k: int, what: str):
    import torch
    global _MinimalToMaximal, _MaximalToMinimal
    if _MinimalToMaximal is None:
        _MinimalToMaximal, _MaximalToMinimal = _map_functions()
    if not torch.is_tensor(a) or a.dtype != torch.float64 or not a.is_cuda:
        raise ValueError(f"{what}: a float64 CUDA tensor expected")
    if a.dim() < 1 or a.shape[-1] != k or a.numel() == 0:
        raise ValueError(f"{what}: [..., {k}] expected, got {tuple(a.shape)}")
    return _stepper(mechanism, 1, a.device.index if a.device.index is not None else torch.cuda.current_device())


def minimal_to_maximal(mechanism: Mechanism, X):
    """minimal_to_maximal on the current torch stream, differentiable: X [..., 2nu] -> Z [..., 13Nb] (CUDA float64).  The backward pass
    maps the quaternion cotangents to the attitude packing (to_attitude) and applies N(z)' (dojo_minimal_to_maximal_vjp_async).
    Once differentiable."""
    s = _map_inputs(mechanism, X, 2 * mechanism.nu, "minimal_to_maximal")
    return _MinimalToMaximal.apply(X, s)


def maximal_to_minimal(mechanism: Mechanism, Z):
    """maximal_to_minimal on the current torch stream, differentiable: Z [..., 13Nb] -> X [..., 2nu] (CUDA float64).  The backward pass
    applies M(z)' (dojo_maximal_to_minimal_vjp_async) and returns the quaternion part as G(q) phibar (from_attitude), tangent to the unit
    sphere as in rollout().  Once differentiable."""
    s = _map_inputs(mechanism, Z, mechanism.nz, "maximal_to_minimal")
    return _MaximalToMinimal.apply(Z, s)


def rollout_minimal(mechanism: Mechanism, X0, U, opts=None):
    """rollout() in minimal coordinates: maximal_to_minimal(rollout(minimal_to_maximal(X0), U)), differentiable with respect to
    X0 [B, 2nu] and U [T, B, nu].  Returns (X_traj [T+1, B, 2nu], status [T, B]).  The gradients are the exact derivative of this
    computation: one maximal rollout from minimal_to_maximal(X0), read out through maximal_to_minimal."""
    Z_traj, status = rollout(mechanism, minimal_to_maximal(mechanism, X0), U, opts)
    return maximal_to_minimal(mechanism, Z_traj), status


def _feedback_function():
    import torch

    class RolloutFeedback(torch.autograd.Function):
        @staticmethod
        def forward(ctx, Z0, K, u_ref, x_ref, K_i, xi0, stepper, opts, T, steps, envs):
            B, dev, nu = Z0.shape[0], Z0.device, stepper.nu
            nx = 2 * nu

            def lay(a, tail, mat):  # [steps, envs, *tail] contiguous; matrices column-major per entry
                if a is None:
                    return None
                a = a.detach()
                a = a.reshape((1, 1) + tail) if a.dim() == len(tail) else (a.unsqueeze(0) if a.dim() == len(tail) + 1 else a)
                a = a.expand((steps, envs) + tail)
                return (a.transpose(-1, -2) if mat else a).contiguous()

            Kc, Kic = lay(K, (nu, nx), True), lay(K_i, (nu, nx), True)
            xrc, urc = lay(x_ref, (nx,), False), lay(u_ref, (nu,), False)
            f64 = dict(dtype=torch.float64, device=dev)
            xi = None if K_i is None else (torch.zeros((B, nx), **f64) if xi0 is None else xi0.detach().expand(B, nx).contiguous().clone())
            Z_traj, X_traj = torch.empty((T + 1, B, stepper.nz), **f64), torch.empty((T + 1, B, nx), **f64)
            Xi = None if K_i is None else torch.empty((T, B, nx), **f64)
            Ua, tape = torch.empty((T, B, nu), **f64), torch.empty((T, B, stepper.nres), **f64)
            p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
            stream = torch.cuda.current_stream(dev).cuda_stream
            stepper.rollout_feedback_tape_device(Z0.detach().contiguous().data_ptr(), Z_traj.data_ptr(), X_traj.data_ptr(), Ua.data_ptr(),
                                                 tape.data_ptr(), B, T, Kc.data_ptr(), steps=steps, envs=envs, dK_i=p(Kic), dx_ref=p(xrc),
                                                 du_ref=p(urc), dxi=p(xi), dXi_traj=p(Xi), opts=opts, stream=stream)
            ctx.save_for_backward(Z_traj, X_traj, Ua, tape, Kc, Kic, xrc, urc, Xi)
            ctx.stepper, ctx.steps, ctx.envs = stepper, steps, envs
            ctx.shapes = [None if a is None else a.shape for a in (K, u_ref, x_ref, K_i, xi0)]
            return Z_traj, X_traj, Ua

        @staticmethod
        def backward(ctx, gZ_traj, gX_traj, gUa):
            Z_traj, X_traj, Ua, tape, Kc, Kic, xrc, urc, Xi = ctx.saved_tensors
            s, steps = ctx.stepper, ctx.steps
            T, B = tape.shape[0], tape.shape[1]
            nu, nx, dev = s.nu, 2 * s.nu, Z_traj.device
            f64 = dict(dtype=torch.float64, device=dev)
            gZ = None if gZ_traj is None else to_attitude(Z_traj, gZ_traj.to(torch.float64)).contiguous()
            gX = None if gX_traj is None else gX_traj.to(torch.float64).contiguous()
            gU = None if gUa is None else gUa.to(torch.float64).contiguous()
            shp = dict(zip(("K", "u_ref", "x_ref", "K_i", "xi0"), ctx.shapes))
            gK = torch.empty((steps, B, nx, nu), **f64) if ctx.needs_input_grad[1] else None
            gur = torch.empty((steps, B, nu), **f64) if ctx.needs_input_grad[2] else None
            gxr = torch.empty((steps, B, nx), **f64) if ctx.needs_input_grad[3] else None
            gKi = torch.empty((steps, B, nx, nu), **f64) if ctx.needs_input_grad[4] else None
            gZ0 = torch.empty((B, s.ngrad), **f64)
            gxi0 = None if Kic is None else torch.empty((B, nx), **f64)
            p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
            stream = torch.cuda.current_stream(dev).cuda_stream
            s.rollout_feedback_vjp_device(Z_traj.data_ptr(), X_traj.data_ptr(), Ua.data_ptr(), tape.data_ptr(), gZ0.data_ptr(), B, T, Kc.data_ptr(),
                                          steps=steps, envs=ctx.envs, dK_i=p(Kic), dx_ref=p(xrc), du_ref=p(urc), dXi_traj=p(Xi), dgZ=p(gZ),
                                          dgX=p(gX), dgU=p(gU), dgK=p(gK), dgK_i=p(gKi), dgx_ref=p(gxr), dgu_ref=p(gur), dgxi0=p(gxi0),
                                          stream=stream)

            def fit(g, name, mat):  # per-environment [steps, B, ...] -> the input's shape, broadcast dimensions summed
                if g is None or shp[name] is None:
                    return None
                g = g.transpose(-1, -2) if mat else g
                n = len(shp[name]) - (2 if mat else 1)  # leading (step / environment) axes of the input
                if n == 0:
                    return g.sum(dim=(0, 1))
                if n == 1:
                    return g.sum(dim=0)
                return g.sum(dim=1, keepdim=True) if shp[name][1] == 1 else g

            gxi = None
            if gxi0 is not None and ctx.needs_input_grad[5]:
                gxi = gxi0.sum(dim=0) if len(shp["xi0"]) == 1 else gxi0
            return (from_attitude(Z_traj[0], gZ0), fit(gK, "K", True), fit(gur, "u_ref", False), fit(gxr, "x_ref", False), fit(gKi, "K_i", True),
                    gxi, None, None, None, None, None)

    return RolloutFeedback


_RolloutFeedback = None


def rollout_feedback(mechanism: Mechanism, Z0, K, u_ref=None, x_ref=None, K_i=None, xi0=None, opts=None, T=None):
    """T closed-loop steps of B environments under u_t = u_ref - K (x_t - x_ref) - K_i xi_t (dojo_rollout_feedback's law),
    differentiable with respect to Z0 [B, 13Nb], K, u_ref, x_ref, K_i and xi0 (CUDA float64 tensors on one device).  Each law tensor
    is [*tail], [B, *tail] or [T, 1 or B, *tail] (tail: [nu, 2nu] for K / K_i, [nu] for u_ref, [2nu] for x_ref); xi0 [2nu] or [B, 2nu]
    (zero when None).  T is taken from a tensor with a step axis, else it must be given.  Returns (Z_traj [T+1, B, 13Nb], X_traj
    [T+1, B, 2nu] (the law's x_t; slab T = maximal_to_minimal(z_T)), U_applied [T, B, nu]).  The backward pass maps the quaternion
    cotangents of Z_traj as rollout() does and returns each input's gradient summed over its broadcast dimensions."""
    import torch
    global _RolloutFeedback
    if _RolloutFeedback is None:
        _RolloutFeedback = _feedback_function()
    nu = mechanism.nu
    tails = {"K": (nu, 2 * nu), "u_ref": (nu,), "x_ref": (2 * nu,), "K_i": (nu, 2 * nu)}
    given = {k: a for k, a in zip(tails, (K, u_ref, x_ref, K_i)) if a is not None}
    for a in list(given.values()) + [Z0] + ([xi0] if xi0 is not None else []):
        if not torch.is_tensor(a) or a.dtype != torch.float64 or not a.is_cuda or a.device != Z0.device:
            raise ValueError("rollout_feedback: Z0 and the law's tensors must be float64 CUDA tensors on one device")
    B = Z0.shape[0]
    steps, envs = 1, 1
    for k, a in given.items():
        n = a.dim() - len(tails[k])
        if n not in (0, 1, 2) or tuple(a.shape[n:]) != tails[k] or (n == 1 and a.shape[0] != B) or (n == 2 and a.shape[1] not in (1, B)):
            raise ValueError(f"rollout_feedback: {k} of shape {tuple(a.shape)}")
        if n == 2:
            if T is not None and a.shape[0] != T:
                raise ValueError(f"rollout_feedback: {k} has {a.shape[0]} steps, T = {T}")
            T, steps = a.shape[0], a.shape[0]
        if (n == 1) or (n == 2 and a.shape[1] == B):
            envs = B
    if T is None:
        raise ValueError("rollout_feedback: T is required when no law tensor has a step axis")
    s = _stepper(mechanism, B, Z0.device.index if Z0.device.index is not None else torch.cuda.current_device())
    return _RolloutFeedback.apply(Z0, K, u_ref, x_ref, K_i, xi0, s, opts, int(T), steps, envs)
