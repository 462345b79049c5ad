// dojo_kin.cuh -- minimal <-> maximal coordinate maps on the device (SURVEY.md 8 f1: the step either side of step! for
// every DojoEnvironments call, simulation/step.jl:42-61).
//
//   minimal_to_maximal   mechanism/state.jl:9-22  ->  set_minimal_coordinates_velocities!  joints/minimal.jl:148-203
//   maximal_to_minimal   mechanism/state.jl:44-66 ->  minimal_coordinates / minimal_velocities
//                        (translational/minimal.jl:57-59,93-113, rotational/minimal.jl:62-67,103-118)
//
// Minimal state x = per joint, in joint order, [c_tra; c_rot; v_tra; v_rot] (2 * input_dimension(joint) entries), batched
// [2 nu x B] like every other array of the ABI.  One THREAD per environment: a map is a few hundred flops per joint and
// the tree is walked root -> leaves (the child state needs the parent's), so there is nothing to share between lanes;
// the kernels are bound by their (tiny) HBM traffic: 8 (2 nu + 13 Nb) bytes per environment.
#pragma once
#include "dojo_math.cuh"
#include "dojo_plan.h"

namespace dj {

struct KinArgs {
  const JointDev* joints;  // plan blob (global memory)
  const int* order;        // joints root -> leaves
  int Ne, Nb, nu, B;
  double h;
  const double* in;
  double* out;
};

struct BodyState { V3 x, v, w; Quat q; };

DJ_DEV BodyState kin_load(const double* z, int b) {
  BodyState s;
  if (b < 0) { s.x = s.v = s.w = v3zero(); s.q = Quat{1.0, 0.0, 0.0, 0.0}; return s; }  // origin (bodies/origin.jl)
  const double* p = z + 13 * b;
  s.x = v3(p[0], p[1], p[2]); s.v = v3(p[3], p[4], p[5]); s.q = Quat{p[6], p[7], p[8], p[9]}; s.w = v3(p[10], p[11], p[12]);
  return s;
}
DJ_DEV Quat axis_angle_to_quaternion(V3 x) {  // orientation/axis_angle.jl:1-11
  const double th = sqrt(dot(x, x));
  if (th > 0.0) { const double s = sin(0.5 * th) / th; return Quat{cos(0.5 * th), s * x.x, s * x.y, s * x.z}; }
  return Quat{1.0, 0.0, 0.0, 0.0};
}
DJ_DEV V3 qrot(V3 v, Quat q) { return rotmat(q) * v; }                            // vector_rotate, rotate.jl:2-5
DJ_DEV Quat next_orientation(Quat q, V3 w, double h) { return qmul(q, qmap(w, h)); }  // integrators/integrator.jl:15
DJ_DEV V3 masked_sum(const double* A, int n, const double* c) {                   // A' * c, A = nullspace mask rows
  V3 r = v3zero();
  for (int i = 0; i < n; ++i) r += c[i] * v3(A[3 * i], A[3 * i + 1], A[3 * i + 2]);
  return r;
}

// one environment: minimal x [2 nu] -> maximal z [13 Nb] (called by one thread)
DJ_DEV void min_to_max_one(const JointDev* joints, const int* order, int Ne, double h, const double* x, double* z) {
  for (int k = 0; k < Ne; ++k) {
    const JointDev& jd = joints[order[k]];
    const int nt = jd.nfree_t, nr = jd.nfree_r, nuj = nt + nr;
    const double* xm = x + 2 * jd.u_off;
    const BodyState pa = kin_load(z, jd.parent);  // written earlier by this thread (root -> leaves)
    const V3 dx = masked_sum(jd.At, nt, xm), dth = masked_sum(jd.Ar, nr, xm + nt);
    const V3 dv = masked_sum(jd.At, nt, xm + nuj), dw = masked_sum(jd.Ar, nr, xm + nuj + nt);
    const Quat qoff = Quat{jd.qoff[0], jd.qoff[1], jd.qoff[2], jd.qoff[3]};
    const V3 va = v3(jd.pa[0], jd.pa[1], jd.pa[2]), vb = v3(jd.pb[0], jd.pb[1], jd.pb[2]);
    // positions
    const Quat dq = axis_angle_to_quaternion(dth);
    const Quat qb = qmul(qmul(pa.q, qoff), dq);
    const V3 xb = pa.x + qrot(va + dx, pa.q) - qrot(vb, qb);
    // previous configuration of the parent, finite-difference configuration of the child
    const V3 xa1 = pa.x - h * pa.v;
    const Quat qa1 = next_orientation(pa.q, -pa.w, h);
    const V3 dx1 = dx - h * dv;
    const Quat dq1 = qmul(dq, qinv(axis_angle_to_quaternion(h * dw)));
    const Quat qb1 = qmul(qmul(qa1, qoff), dq1);
    const V3 xb1 = xa1 + qrot(va + dx1, qa1) - qrot(vb, qb1);
    // finite-difference velocities
    const V3 vel = (1.0 / h) * (xb - xb1);
    const V3 om = (2.0 / h) * qvec(qmul(qconj(qb1), qb));  // angular_velocity, integrator.jl:22-24
    double* o = z + 13 * jd.child;
    o[0] = xb.x; o[1] = xb.y; o[2] = xb.z; o[3] = vel.x; o[4] = vel.y; o[5] = vel.z;
    o[6] = qb.s; o[7] = qb.x; o[8] = qb.y; o[9] = qb.z; o[10] = om.x; o[11] = om.y; o[12] = om.z;
  }
}

// translational displacement in the parent frame (translational/minimal.jl:4-12)
DJ_DEV V3 tra_displacement(const JointDev& jd, V3 xa, Quat qa, V3 xb, Quat qb) {
  const V3 d = xb + qrot(v3(jd.pb[0], jd.pb[1], jd.pb[2]), qb) - xa - qrot(v3(jd.pa[0], jd.pa[1], jd.pa[2]), qa);
  return tmul(rotmat(qa), d);
}

DJ_DEV void min_to_max_env(const KinArgs& a, int e) {
  min_to_max_one(a.joints, a.order, a.Ne, a.h, a.in + (size_t)e * 2 * a.nu, a.out + (size_t)e * 13 * a.Nb);
}

// one joint: maximal z [13 Nb] -> its slice of the minimal x [2 nu].  Reads only the joint's parent and child bodies, so the joints of
// one environment may be mapped in any order or in parallel (one lane per joint: the feedback stage of dojo_step_kernel<..., FB>)
DJ_DEV void max_to_min_joint(const JointDev& jd, double h, const double* z, double* x) {
  const int nt = jd.nfree_t, nr = jd.nfree_r, nuj = nt + nr;
  if (nuj == 0) return;
  double* xm = x + 2 * jd.u_off;
  const BodyState A = kin_load(z, jd.parent), Bc = kin_load(z, jd.child);
  const Quat qoffi = qinv(Quat{jd.qoff[0], jd.qoff[1], jd.qoff[2], jd.qoff[3]});
  // one step backward in time
  const V3 xa1 = A.x - h * A.v, xb1 = Bc.x - h * Bc.v;
  const Quat qa1 = next_orientation(A.q, -A.w, h), qb1 = next_orientation(Bc.q, -Bc.w, h);
  const V3 et = tra_displacement(jd, A.x, A.q, Bc.x, Bc.q);
  const V3 et1 = tra_displacement(jd, xa1, qa1, xb1, qb1);
  const Quat q = qmul(qmul(qoffi, qinv(A.q)), Bc.q);
  const Quat q1 = qmul(qmul(qoffi, qinv(qa1)), qb1);
  const V3 th = rotation_vector(q);
  const V3 dth = (1.0 / h) * rotation_vector(qmul(qinv(q1), q));
  const V3 det = (1.0 / h) * (et - et1);
  for (int i = 0; i < nt; ++i) {
    const V3 ai = v3(jd.At[3 * i], jd.At[3 * i + 1], jd.At[3 * i + 2]);
    xm[i] = dot(ai, et);
    xm[nuj + i] = dot(ai, det);
  }
  for (int i = 0; i < nr; ++i) {
    const V3 ai = v3(jd.Ar[3 * i], jd.Ar[3 * i + 1], jd.Ar[3 * i + 2]);
    xm[nt + i] = dot(ai, th);
    xm[nuj + nt + i] = dot(ai, dth);
  }
}

// one environment: maximal z [13 Nb] -> minimal x [2 nu]
DJ_DEV void max_to_min_one(const JointDev* joints, int Ne, double h, const double* z, double* x) {
  for (int j = 0; j < Ne; ++j) max_to_min_joint(joints[j], h, z, x);
}

DJ_DEV void max_to_min_env(const KinArgs& a, int e) {
  max_to_min_one(a.joints, a.Ne, a.h, a.in + (size_t)e * 13 * a.Nb, a.out + (size_t)e * 2 * a.nu);
}

// the map kernels belong to the main compilation (dojo_b200.cu); dojo_b200_cm.cu includes this header for max_to_min_joint only
#if defined(__CUDACC__) && !defined(DJ_ANY_CONTACT)
__global__ void dojo_min_to_max_kernel(const KinArgs a) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < a.B) min_to_max_env(a, e);
}
__global__ void dojo_max_to_min_kernel(const KinArgs a) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < a.B) max_to_min_env(a, e);
}
#endif

}  // namespace dj
