"""M(z)' gX and N(z)' gZ on the CPU -- TEST INFRASTRUCTURE for tests/test_minimal_vjp.py.

hostcheck_map_vjp runs exactly the per-state device routines of dojo_maximal_to_minimal_vjp / dojo_minimal_to_maximal_vjp
(dojo_kinjac.cuh: max_to_min_vjp_env, min_to_max_vjp_env) with one "thread", so that they can be compared with the dense
maximal_to_minimal_jacobian / minimal_to_maximal_jacobian of hostcheck.cpp.  The entry is appended to hostcheck.cpp in a translation
unit of its own and compiled into a library of its own.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from .harness import HERE, HostCheck, _d, _dp

ENTRY = r"""
// mode 0: out [B][12 Nb] = M(z)' in [B][2 nu];  mode 1: out [B][2 nu] = N(z)' in [B][12 Nb]
extern "C" void hostcheck_map_vjp(void* p, int mode, int B, const double* Z, const double* in, double* out) {
  Mech* m = static_cast<Mech*>(p);
  MapVjpArgs a;
  std::memset(&a, 0, sizeof(a));
  a.joints = m->joints.data(); a.order = m->order.data();
  a.Ne = m->Ne; a.Nb = m->Nb; a.nu = m->nu; a.n = B; a.h = m->h;
  a.Z = Z; a.in = in; a.out = out;
  std::vector<double> ws(mode == 0 ? (size_t)24 * m->Ne : min_to_max_vjp_ws_doubles(m->Nb));
  for (int e = 0; e < B; ++e) {
    if (mode == 0) max_to_min_vjp_env(a, e, ws.data(), 0, 1, [] {});
    else min_to_max_vjp_env(a, e, ws.data(), 0, 1, [] {});
  }
}
"""
LIB = os.path.join(HERE, "_build", "libdojo_hostcheck_minvjp.so")


def build() -> str:
    src = os.path.join(HERE, "hostcheck.cpp")
    deps = [src, __file__] + [os.path.join(HERE, "..", "..", "dojo.jl_b200", "csrc", f) for f in ("dojo_kinjac.cuh", "dojo_kin.cuh", "dojo_math.cuh")]
    if os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in deps):
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    tu = os.path.join(os.path.dirname(LIB), "hostcheck_minvjp.cpp")
    with open(tu, "w") as f:
        f.write(f'#include "{src}"\n' + ENTRY)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-o", LIB + ".tmp", tu])
    os.replace(LIB + ".tmp", LIB)
    return LIB


class MapVjp(HostCheck):
    """HostCheck's maps and Jacobians plus the adjoints of the maps, from the library of build()"""

    def __init__(self, mech):
        from . import harness
        old = harness.build
        harness.build = build  # HostCheck loads harness.build()'s library; this one is a superset of it
        try:
            super().__init__(mech)
        finally:
            harness.build = old
        self.L.hostcheck_map_vjp.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp, _dp, _dp]

    def _run(self, mode, Z, g, nout):
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=float)
        g = np.ascontiguousarray(np.atleast_2d(g), dtype=float)
        out = np.full((Z.shape[0], nout), np.nan)
        self.L.hostcheck_map_vjp(self.h, mode, Z.shape[0], _d(Z), _d(g), _d(out))
        return out

    def max_to_min_vjp(self, Z, gX):
        """[B, 12Nb] = M(z)' gX per state"""
        return self._run(0, Z, gX, self.ns)

    def min_to_max_vjp(self, Z, gZ):
        """[B, 2nu] = N(z)' gZ per state, Z = minimal_to_maximal(X)"""
        return self._run(1, Z, gZ, self.nm)
