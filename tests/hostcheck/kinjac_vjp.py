"""M(z)' w on the CPU -- TEST INFRASTRUCTURE for tests/test_rollout_feedback_vjp.py.

hostcheck_max_to_min_vjp runs exactly the device routines of the closed-loop adjoint (dojo_kinjac.cuh: max_to_min_vjp_joint per joint,
then max_to_min_vjp_fold per body) with one "thread", so that they can be compared with the dense maximal_to_minimal_jacobian of
hostcheck.cpp.  The entry is appended to hostcheck.cpp in a translation unit of its own and compiled into a library of its own.
"""
import ctypes as C
import os
import subprocess

import numpy as np

import dojo_jl_b200 as dj
from .harness import HERE, HostCheck, _d, _dp

ENTRY = r"""
extern "C" void hostcheck_max_to_min_vjp(void* p, int B, const double* Z, const double* W, double* G) {
  Mech* m = static_cast<Mech*>(p);
  std::vector<double> s((size_t)24 * m->Ne, 0.0);
  for (int e = 0; e < B; ++e) {
    const double* z = Z + (size_t)e * 13 * m->Nb;
    for (int j = 0; j < m->Ne; ++j) {
      const JointDev& jd = m->joints[j];
      if (jd.nfree_t + jd.nfree_r > 0)
        max_to_min_vjp_joint(jd, kin_load(z, jd.parent), kin_load(z, jd.child), m->h, W + (size_t)e * 2 * m->nu + 2 * jd.u_off, s.data() + 24 * j);
    }
    for (int b = 0; b < m->Nb; ++b) max_to_min_vjp_fold(m->joints.data(), m->Ne, b, s.data(), G + ((size_t)e * m->Nb + b) * 12);
  }
}
"""
LIB = os.path.join(HERE, "_build", "libdojo_hostcheck_vjp.so")


def build() -> str:
    src = os.path.join(HERE, "hostcheck.cpp")
    deps = [src, __file__] + [os.path.join(HERE, "..", "..", "dojo.jl_b200", "csrc", f) for f in ("dojo_kinjac.cuh", "dojo_kin.cuh", "dojo_math.cuh")]
    if os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in deps):
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    tu = os.path.join(os.path.dirname(LIB), "hostcheck_vjp.cpp")
    with open(tu, "w") as f:
        f.write(f'#include "{src}"\n' + ENTRY)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-o", LIB + ".tmp", tu])
    os.replace(LIB + ".tmp", LIB)
    return LIB


class KinJacVjp(HostCheck):
    """HostCheck's maps and Jacobians plus M(z)' w, from the library of build()"""

    def __init__(self, mech):
        from . import harness
        old = harness.build
        harness.build = build  # HostCheck loads harness.build()'s library; this one is a superset of it
        try:
            super().__init__(mech)
        finally:
            harness.build = old
        self.L.hostcheck_max_to_min_vjp.argtypes = [C.c_void_p, C.c_int, _dp, _dp, _dp]

    def max_to_min_vjp(self, Z, W):
        """[B, 12Nb] = M(z)' w per environment"""
        Z = np.ascontiguousarray(np.atleast_2d(Z), dtype=float)
        W = np.ascontiguousarray(np.atleast_2d(W), dtype=float)
        G = np.empty((Z.shape[0], self.ns))
        self.L.hostcheck_max_to_min_vjp(self.h, Z.shape[0], _d(Z), _d(W), _d(G))
        return G


def mechanisms():
    """(name, mechanism) for every mechanism in dojo.jl_b200/mechanisms/ and the two-body snake of each of the 16 joint prototypes"""
    from test_joint_prototypes import PROTOTYPES, snake
    mdir = os.path.join(os.path.dirname(dj.__file__), "mechanisms")
    out = [(f[:-5], dj.get_mechanism(f[:-5])) for f in sorted(os.listdir(mdir)) if f.endswith(".json")]
    return out + [(f"snake_{t}", snake(t)) for t in PROTOTYPES]
