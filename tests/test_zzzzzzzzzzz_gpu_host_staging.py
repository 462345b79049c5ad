"""Pointer kinds of the synchronous C-ABI entries on the H100, and the reuse of the handle's staging arena.

Every synchronous entry takes host or device pointers.  For each entry this file calls the C function with pageable numpy buffers,
page-locked numpy buffers (torch pin_memory) and torch CUDA tensors, and, where an *_async form exists, that form on a torch stream;
every output must be bit-identical across the kinds, including the parts of the output buffers the entry leaves untouched (every output
starts from the same fill pattern).  Optional outputs passed as null must leave the others unchanged.  Host-pointer calls share one
grow-only staging arena per handle: a sequence of calls whose sizes grow and shrink must give, call by call, what a fresh handle gives.
"""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from dojo_jl_b200 import capi
from dojo_jl_b200 import environments as E
from dojo_jl_b200.solver import BatchedStepper, cost_arrays, feedback_arrays
from test_rollout_vjp import _mech, _start

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

KINDS = ("pageable", "pinned", "device")
FILL = {np.float64: -1234.5, np.int32: -7}


class Out:
    """an output array of the call, filled with FILL before the call"""
    def __init__(self, *shape, dtype=np.float64):
        self.shape, self.dtype = shape, dtype


class Host:
    """an input the entry reads on the host whatever the pointer kind (dojo_env_policy_rollout's mean / std)"""
    def __init__(self, a):
        self.a = a


class Struct:
    """a DojoFeedback / DojoQuadraticCost whose arrays take the call's pointer kind"""
    def __init__(self, cls, steps, envs, *arrays):
        self.cls, self.steps, self.envs, self.arrays = cls, steps, envs, arrays


def _buffer(kind, a, keep):
    if kind == "device":
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        keep.append(t)
        return C.c_void_p(t.data_ptr()), lambda: t.cpu().numpy()
    if kind == "pinned":
        t = torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
        keep.append(t)
        n = t.numpy()
    else:
        n = np.array(a, copy=True, order="C")
    keep.append(n)
    return C.c_void_p(n.ctypes.data), lambda: n.copy()


def call(s, kind, name, args, async_args=None):
    """Calls `name` (or, kind "async", name + "_async" with async_args(args) + the stream) and returns the outputs in argument order."""
    keep, reads, cargs = [], [], []
    buf_kind = "device" if kind == "async" else kind
    for a in args:
        if isinstance(a, Out):
            p, read = _buffer(buf_kind, np.full(a.shape, FILL[a.dtype], dtype=a.dtype), keep)
            cargs.append(p)
            reads.append(read)
        elif isinstance(a, np.ndarray):
            cargs.append(_buffer(buf_kind, a, keep)[0])
        elif isinstance(a, Host):
            cargs.append(_buffer("pageable", a.a, keep)[0])
        elif isinstance(a, Struct):
            ptrs = [None if x is None else C.cast(_buffer(buf_kind, x, keep)[0], C.POINTER(C.c_double)) for x in a.arrays]
            st = a.cls(a.steps, a.envs, *ptrs)
            keep.append(st)
            cargs.append(C.byref(st))
        else:
            cargs.append(a)
    torch.cuda.synchronize()
    if kind == "async":
        stream = torch.cuda.Stream()
        with torch.cuda.stream(stream):
            rc = getattr(s.L, name + "_async")(*(async_args or (lambda x: x))(cargs), C.c_void_p(stream.cuda_stream))
        stream.synchronize()
    else:
        rc = getattr(s.L, name)(*cargs)
    assert rc == 0, (name, kind, s.L.dojo_last_error(s.h))
    return [r() for r in reads]


def same(a, b, what):
    assert len(a) == len(b), what
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), f"{what}: output {i}"


def check(s, name, args, has_async=True, async_args=None, optional=()):
    """pointer kinds (and the async form) agree; each index in `optional` replaced by null leaves the other outputs unchanged"""
    ref = call(s, "pageable", name, args)
    for kind in KINDS[1:] + (("async",) if has_async else ()):
        same(call(s, kind, name, args, async_args), ref, f"{name} {kind}")
    outs = [i for i, a in enumerate(args) if isinstance(a, Out)]
    for i in optional:
        kept = [k for k, j in enumerate(outs) if j != i]
        for kind in KINDS:
            got = call(s, kind, name, [None if j == i else a for j, a in enumerate(args)])
            same(got, [ref[k] for k in kept], f"{name} {kind} without argument {i}")
    return ref


def _stepper(name, B):
    m = _mech(name)
    return m, BatchedStepper(m, B, 0)


def opts():
    return C.byref(capi.solver_options())


def test_rollout_step_and_record_entries():
    B, T = 48, 5
    m, s = _stepper("ant", B)
    Z0, U = _start(m, B, T, 3)
    o = opts()
    check(s, "dojo_rollout", [s.h, o, B, T, Z0, U, Out(B, m.nz), Out(T, B, m.nz), Out(B, dtype=np.int32)], optional=(7, 8))
    check(s, "dojo_rollout", [s.h, o, B, T, Z0, None, Out(B, m.nz), None, Out(B, dtype=np.int32)])
    check(s, "dojo_step_record", [s.h, o, B, Z0, U[0], Out(B, m.nz), Out(B, 12 * m.Nb), Out(B, 8), Out(B, dtype=np.int32),
                                  Out(B, dtype=np.int32)], optional=(8, 9))
    check(s, "dojo_simulate_record", [s.h, o, B, T, Z0, U, Out(B, m.nz), Out(T, B, m.nz), Out(T, B, 12 * m.Nb), Out(T, B, 8),
                                      Out(B, dtype=np.int32)], has_async=False, optional=(7, 8, 9, 10))
    s.close()


def test_step_grad_uses_both_chunk_buffers():
    """B above the gradient chunk (128 MB of Jacobians): the host path alternates the two chunk buffers and their copy stream"""
    m = _mech("atlas")
    ng = 12 * m.Nb
    B = 2 * max(1, (128 << 20) // ((ng * ng + ng * m.nu) * 8)) + 3
    s = BatchedStepper(m, B, 0)
    Z0, U = _start(m, B, 1, 5)
    check(s, "dojo_step_grad", [s.h, opts(), B, Z0, U[0], None, Out(B, m.nz), Out(B, ng, ng), Out(B, ng, m.nu), Out(B, dtype=np.int32),
                                Out(B, dtype=np.int32), 0], optional=(9, 10))
    s.close()


def test_step_grad_contact():
    B = 24
    m, s = _stepper("quadruped", B)
    Z0, U = _start(m, B, 1, 7)
    ng = 12 * m.Nb
    args = [s.h, opts(), B, Z0, U[0], Out(B, m.nz), Out(B, ng, ng), Out(B, ng, m.nu), Out(B, ng, 5 * m.Ni), Out(B, dtype=np.int32),
            Out(B, dtype=np.int32)]
    check(s, "dojo_step_grad_contact", args, async_args=lambda a: a[:5] + [None] + a[5:] + [0], optional=(9, 10))
    s.close()


def test_minimal_coordinate_entries():
    B = 32
    m, s = _stepper("quadruped", B)
    Z0, U = _start(m, B, 1, 9)
    X = s.maximal_to_minimal(Z0)
    nm = 2 * m.nu
    check(s, "dojo_maximal_to_minimal", [s.h, B, Z0, Out(B, nm)])
    check(s, "dojo_minimal_to_maximal", [s.h, B, X, Out(B, m.nz)])
    check(s, "dojo_maximal_to_minimal_jacobian", [s.h, B, Z0, Out(B, 12 * m.Nb, nm)])
    check(s, "dojo_step_minimal_flags", [s.h, opts(), B, X, U[0], Out(B, nm), Out(B, dtype=np.int32), Out(B, dtype=np.int32), 0],
          has_async=False, optional=(6, 7))
    check(s, "dojo_minimal_gradients", [s.h, opts(), B, X, U[0], Out(B, nm), Out(B, nm, nm), Out(B, nm, m.nu), Out(B, dtype=np.int32),
                                        Out(B, dtype=np.int32)], has_async=False, optional=(8, 9))
    s.close()


def test_trajectory_entries():
    """the entries whose own tests compare pointer kinds, once each, through the same harness"""
    B, T = 16, 4
    m, s = _stepper("ant", B)
    Z0, U = _start(m, B, T, 11)
    X0 = s.maximal_to_minimal(Z0)
    ng, nm, o = 12 * m.Nb, 2 * m.nu, opts()
    i32 = dict(dtype=np.int32)
    check(s, "dojo_rollout_grad", [s.h, o, B, T, Z0, U, Out(T + 1, B, m.nz), Out(T, B, ng, ng), Out(T, B, ng, m.nu), Out(T, B, **i32),
                                   Out(T, B, **i32)], optional=(9, 10))
    check(s, "dojo_rollout_minimal_gradients", [s.h, o, B, T, X0, U, Out(T + 1, B, nm), Out(T, B, nm, nm), Out(T, B, nm, m.nu),
                                                Out(T, B, **i32), Out(T, B, **i32)], has_async=False, optional=(9, 10))
    traj, tape, _, _ = check(s, "dojo_rollout_tape", [s.h, o, B, T, Z0, U, Out(T + 1, B, m.nz), Out(T, B, m.nres), Out(T, B, **i32),
                                                      Out(T, B, **i32)], optional=(8, 9))
    gZ = np.random.default_rng(12).normal(size=(T + 1, B, ng))
    check(s, "dojo_rollout_vjp", [s.h, B, T, traj, U, tape, gZ, Out(B, ng), Out(T, B, m.nu), Out(B, **i32)], optional=(8, 9))
    K = np.random.default_rng(13).normal(0.0, 0.1, (m.nu, nm))
    steps, envs, Kc, xr, ur, Ki = feedback_arrays(T, B, m.nu, K, x_ref=X0[0], K_i=0.1 * K)
    fb = Struct(capi.DojoFeedback, steps, envs, Kc, Ki, xr, ur)
    check(s, "dojo_rollout_feedback", [s.h, o, B, T, Z0, fb, np.zeros((B, nm)), Out(B, m.nz), Out(T, B, m.nz), Out(T, B, m.nu), Out(B, **i32)],
          optional=(8, 9, 10))
    Xt, Gx, Gu, _, _ = s.rollout_minimal_gradients(X0, U, T)
    cost = Struct(capi.DojoQuadraticCost, *cost_arrays(T, B, m.nu, np.eye(nm), 0.1 * np.eye(m.nu), x_goal=X0[0]))
    check(s, "dojo_lqr_backward", [s.h, B, T, cost, None, Xt, U, Gx, Gu, None, Out(T, B, m.nu, nm), Out(T, B, m.nu), Out(B, 2), Out(B, **i32)],
          optional=(12, 13))
    s.close()


def _env(B):
    env = E.get_environment("ant_ars", batch=B)
    s = BatchedStepper(env.mechanism, B, 0)
    ns, na = s.env_sizes(env.spec)
    Z0, _ = _start(env.mechanism, B, 1, 17)
    S = np.zeros((B, ns))
    S[:, : 2 * env.mechanism.nu] = s.maximal_to_minimal(Z0)
    return env, s, S, ns, na


def test_environment_entries():
    B, T = 24, 4
    env, s, S, ns, na = _env(B)
    rng = np.random.default_rng(19)
    A = rng.uniform(-1, 1, (T, B, na))
    spec, o, i32 = C.byref(env.spec), opts(), dict(dtype=np.int32)
    check(s, "dojo_env_step", [s.h, o, spec, B, S, A[0], Out(B, ns), Out(B), Out(B, **i32), Out(B, **i32), Out(B, **i32)],
          optional=(7, 8, 9, 10))
    check(s, "dojo_env_rollout", [s.h, o, spec, B, T, S, A, Out(B, ns), Out(B), Out(B, **i32)], has_async=False, optional=(8, 9))
    Theta = rng.normal(0.0, 0.05, (B, ns, na))
    mean, std = S.mean(axis=0), S.std(axis=0) + 1.0
    check(s, "dojo_env_policy_rollout", [s.h, o, spec, B, T, S, Theta, Host(mean), Host(std), Out(B, ns), Out(B), Out(B, **i32), Out(T, B, ns)],
          has_async=False, optional=(10, 11, 12))
    s.close()


def test_arena_reuse_matches_fresh_handles():
    """one handle through calls whose staging grows and shrinks gives, call by call, what a fresh handle gives"""
    B = 16
    env = E.get_environment("ant_ars", batch=B)
    m, spec = env.mechanism, env.spec
    Z0, U = _start(m, B, 20, 29)
    probe = BatchedStepper(m, B, 0)
    X0 = probe.maximal_to_minimal(Z0)
    ns, na = probe.env_sizes(spec)
    Xt, Gx, Gu, _, _ = probe.rollout_minimal_gradients(X0, U[:3], 3)
    traj, tape, _, _ = probe.rollout_tape(Z0, U, 20)
    probe.close()
    S = np.zeros((B, ns))
    S[:, : 2 * m.nu] = X0
    rng = np.random.default_rng(23)
    gZ, Theta = rng.normal(size=(6, B, 12 * m.Nb)), rng.normal(0.0, 0.05, (B, na, ns))
    K = rng.normal(0.0, 0.1, (m.nu, 2 * m.nu))
    cost = SimpleNamespace(Q=np.eye(2 * m.nu), R=0.1 * np.eye(m.nu), x_goal=None, u_goal=None, Q_final=None, x_goal_final=None)
    calls = [
        lambda s: s.rollout_tape(Z0, U, 20),
        lambda s: s.lqr_backward(Xt, U[:3], Gx, Gu, cost),
        lambda s: s.rollout_vjp(traj[:6], U[:5], tape[:5], gZ),
        lambda s: [x for x in s.rollout_feedback(Z0, 8, K, x_ref=X0[0], record=True) if x is not None],
        lambda s: s.rollout_grad(Z0, U, 20),
        lambda s: s.env_policy_rollout(spec, S, Theta, 6, record_states=True),
    ]
    shared = BatchedStepper(m, B, 0)
    got = [list(f(shared)) for f in calls]
    shared.close()
    for k, f in enumerate(calls):
        s = BatchedStepper(m, B, 0)
        same(got[k], list(f(s)), f"call {k}")
        s.close()


def test_async_call_then_growing_host_call():
    """an *_async call on a caller stream, immediately followed by a host-pointer call that grows the staging arena"""
    B, T = 32, 3
    m, s = _stepper("ant", B)
    Z0, U = _start(m, B, 40, 31)
    ref_s = BatchedStepper(m, B, 0)
    Zf_ref, st_ref, traj_ref = ref_s.rollout(Z0, U[:T], T, record=True)
    big_ref = ref_s.rollout_tape(Z0, U, 40)
    ref_s.close()
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    dZ0, dU = d(Z0), d(U[:T])
    dZf, dtraj = torch.empty((B, m.nz), dtype=torch.float64, device="cuda"), torch.empty((T, B, m.nz), dtype=torch.float64, device="cuda")
    dst = torch.empty(B, dtype=torch.int32, device="cuda")
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        s.rollout_device(dZ0.data_ptr(), dU.data_ptr(), dZf.data_ptr(), B, T, dtraj=dtraj.data_ptr(), dstatus=dst.data_ptr(), stream=stream.cuda_stream)
    big = s.rollout_tape(Z0, U, 40)  # host pointers: the arena grows while the async rollout may still run
    stream.synchronize()
    same([dZf.cpu().numpy(), dtraj.cpu().numpy(), dst.cpu().numpy()], [Zf_ref, traj_ref, st_ref], "async rollout")
    same(list(big), list(big_ref), "host-pointer tape")
    s.close()
