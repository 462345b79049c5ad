"""The block LDU's flat program (dojo_plan.h LduOp) -- CPU suite.

factorize() and solve() read one 48-byte op per elimination step, in each warp's phase order, instead of walking sched -> ElimStep ->
ElimNb -> ilist.  Two checks:
  * the program the plan builder emits names, for every op, exactly the addresses and bounds the chain yields (every mechanism of
    the package and the 16- / 17- / 32-node boundary shapes of tests/test_shape_boundaries.py);
  * the emulated kernels reproduce, bit for bit, the steps and gradients written by tools/make_ldu_golden.py from the revision
    before the program (tests/golden/ldu_emulation.npz).
"""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import dojo_jl_b200 as dj
from dojo_jl_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MECHS = sorted(f[:-5] for f in os.listdir(os.path.join(ROOT, "dojo.jl_b200", "mechanisms")) if f.endswith(".json"))

# walks the chain the program replaces and counts the ops that differ from it
CHECK = r"""
extern "C" int ldu_program_mismatches(const DojoMechanismDesc* d) {
  EmuHandle* e = static_cast<EmuHandle*>(hostemu_create(d));
  if (!e) return -1;
  const DojoHandle* h = e->h;
  const Plan& P = h->plan;
  const int nw = h->nw;
  const int* cnt = P.sched + P.prog_cnt;
  const LduOp* ops = reinterpret_cast<const LduOp*>(P.sched + P.prog_ops);
  int bad = 0;
  if (P.prog_ops % 4 != 0 || (reinterpret_cast<uintptr_t>(ops) & 15) != 0) bad++;
  for (int w = 0; w < nw; ++w) {
    int k = cnt[P.nphase * nw + w];
    for (int ph = 0; ph < P.nphase; ++ph) {
      const int s0 = P.sched[2 * (ph * nw + w)], sn = P.sched[2 * (ph * nw + w) + 1];
      if (cnt[ph * nw + w] != sn) bad++;
      for (int s = 0; s < sn; ++s, ++k) {
        const ElimStep& st = P.steps[s0 + s];
        const int* w = ops[k].w;
        bool ok = lo16(w[0]) == st.d_off && hi16(w[0]) == st.vec_off && byte_of(w[1], 0) == st.n && byte_of(w[1], 1) == st.nnb &&
                  hi16(w[1]) == st.fold_cnt && lo16(w[2]) == st.fold_off;
        const int fold[kLduFold] = {hi16(w[2]), lo16(w[3]), hi16(w[3])};
        for (int j = 0; j < st.fold_cnt && j < kLduFold; ++j) ok = ok && fold[j] == P.ilist[st.fold_off + j];
        for (int i = 0; i < st.nnb; ++i) {
          const ElimNb& nb = st.nb[i];
          const int* o = w + 4 * (1 + i);
          ok = ok && lo16(o[0]) == nb.L_off && (nb.fwd_abs >= 0 ? hi16(o[0]) == nb.fwd_abs : hi16(o[0]) == kLduNone) && lo16(o[1]) == nb.vec_off &&
               hi16(o[1]) == nb.U_off && byte_of(o[2], 0) == nb.n && byte_of(o[2], 1) == nb.U_row && byte_of(o[2], 2) == nb.U_k && byte_of(o[2], 3) == nb.ld;
          for (int j = 0; j < st.nnb; ++j) ok = ok && (j ? hi16(o[3]) : lo16(o[3])) == st.tgt[i][j];
        }
        if (!ok) bad++;
      }
    }
    // the ops of warp w end where those of warp w + 1 begin
    if (w + 1 < nw && k != cnt[P.nphase * nw + w + 1]) bad++;
  }
  hostemu_destroy(e);
  return bad;
}
"""


@pytest.fixture(scope="module")
def checker():
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from hostemu import gen
    d = tempfile.mkdtemp(prefix="dojo_ldu_")
    src, lib = os.path.join(d, "check.cpp"), os.path.join(d, "libcheck.so")
    with open(src, "w") as f:
        f.write(f'#include "{gen.generate()}"\n#include <cstdint>\n' + CHECK)
    subprocess.check_call(["g++", "-O0", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-w", "-o", lib, src])
    L = C.CDLL(lib)
    L.ldu_program_mismatches.argtypes = [C.POINTER(capi.DojoMechanismDesc)]
    return L


def _shapes():
    """the boundary shapes that build (n33 / c33 are over the size limit); star32 folds 31 children into its root"""
    from test_shape_boundaries import EXPECTED
    return sorted(EXPECTED)


@pytest.mark.parametrize("name", MECHS + ["shape:" + s for s in _shapes()])
def test_program_matches_chain(checker, name):
    if name.startswith("shape:"):
        from test_shape_boundaries import shape
        mech = shape(name[6:])
    else:
        mech = dj.get_mechanism(name)
    desc, keep = capi.flatten(mech)
    assert checker.ldu_program_mismatches(C.byref(desc)) == 0


def test_outputs_match_parent_emulation():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_ldu_golden as g
    ref = np.load(os.path.join(ROOT, "tests", "golden", "ldu_emulation.npz"))
    got = g.generate()
    assert sorted(got) == sorted(ref.files)
    diff = [k for k in ref.files if ref[k].shape != got[k].shape or ref[k].tobytes() != np.asarray(got[k], ref[k].dtype).tobytes()]
    assert not diff, diff
