// dojo_lqr.cuh -- batched Riccati backward pass of time-varying LQR / iLQR in minimal coordinates (dojo_lqr_backward).
//
// One CTA per environment runs t = T-1 ... 0 with P, p and every per-step temporary in dynamic shared memory; A_t = Gx[t, e] and
// B_t = Gu[t, e] are read from global memory once each.  Cost (DojoQuadraticCost, include/dojo_b200.h):
//   l_t = 1/2 (x - xg_t)' Q_t (x - xg_t) + 1/2 (u - ug_t)' R_t (u - ug_t),   l_T = 1/2 (x - xg_T)' Q_f (x - xg_T)
// Recursion (Tassa, Erez, Todorov 2012; K with the sign of the forward law u = u_bar + alpha k - K (x - x_bar)):
//   P_T = Q_f, p_T = Q_f (x_T - xg_T)
//   Qx = Q_t dx + A'p     Qu = R_t du + B'p     Qxx = Q_t + A'PA     Quu = R_t + B'PB     Qux = B'PA
//   K = (Quu + mu I)^-1 Qux,  k = -(Quu + mu I)^-1 Qu               (Cholesky on the active inputs; inactive rows of K and k are 0)
//   P = Qxx + K'Quu K - K'Qux - Qux'K  (symmetrised),  p = Qx - K'Quu k - K'Qu + Qux'k,  dV += [k'Qu, 1/2 k'Quu k]
// Only the active inputs enter: with a = the active index set, B is replaced by B[:, a], Quu by Quu[a, a], Qux by Qux[a, :] and Qu by
// Qu[a] (R's full rows still multiply du), which is the recursion with the inactive inputs held at u_bar.
//
// Every output element is computed by one thread in a fixed order, so the result does not depend on thread scheduling.  The kernel body
// also runs on the CPU emulation of the test suite (tests/hostemu/lqr.py), which rewrites the dynamic shared-memory declaration.
#pragma once
#include "dojo_math.cuh"

namespace dj {

#define DJ_LQR_MAX_NU 64        // bound of LqrArgs::act; the shared-memory working set bounds nu further (lqr_smem_bytes)
#define DJ_LQR_MAX_THREADS 512

struct LqrArgs {
  int nu, B, T, na;            // inputs, environments, steps, active inputs
  int act[DJ_LQR_MAX_NU];      // [na] active input indices, ascending (copied to shared memory by the kernel)
  int steps, envs;             // cost arrays: entry (t, e) at (steps > 1 ? t : 0) * envs + (envs > 1 ? e : 0)
  const double *Q, *R, *xg, *ug, *Qf, *xgf;  // xg, ug, xgf nullable (0)
  const double *X, *U;         // X [2nu x B x (T+1)], U [nu x B x T] nullable (0)
  const double *Gx, *Gu;       // [2nu x 2nu x B x T], [2nu x nu x B x T], pair (t, e) at t * B + e
  const double* mu;            // [B] nullable (0)
  double *K, *k, *dV;          // [nu x 2nu x B x T], [nu x B x T], [2 x B] nullable
  int32_t* status;             // [B] nullable: 0, or t + 1 when the Cholesky of Quu failed at step t
};

// Shared-memory matrices are column-major with an ODD leading dimension (lx = nx + 1 for the nx-row ones, ln = na | 1 for the na-row
// ones): a thread of a product reads down a column while its neighbour reads the next column, ld doubles away, and an odd ld puts the
// 16 doubles of a half-warp in 16 different bank pairs.
DJ_DEV int lqr_odd(int n) { return n | 1; }

// dynamic shared memory of one CTA (nx = 2 nu, lx = nx + 1): three lx x nx matrices, two lx x nu, two (nu + 1) x nx / nu, five vectors,
// the failure flag and the active indices.  Atlas (nu = 36): 202,624 bytes; nu = 38 is the largest that fits the H100's 227 KB opt-in
// maximum per block.
inline size_t lqr_smem_bytes(int nu) {
  const size_t nx = 2 * (size_t)nu, lx = nx + 1, n = nu;
  return (3 * lx * nx + 2 * lx * n + (n + 1) * (nx + n) + 3 * nx + 2 * n + 2) * sizeof(double) + n * sizeof(int);
}

// acc[i][j] += sum_k op(A)(i_i, k) B(k, j_j) over the rows i0, i1 and columns j0, j1 of one thread; op(A) = A' when TA.  Column-major
// operands, fixed summation order.
template <bool TA>
DJ_DEV void lqr_tile(double (&acc)[2][2], const double* A, int lda, const double* Bm, int ldb, int i0, int i1, int j0, int j1, int kd) {
  for (int q = 0; q < kd; ++q) {
    const double a0 = TA ? A[q + (size_t)lda * i0] : A[i0 + (size_t)lda * q];
    const double a1 = TA ? A[q + (size_t)lda * i1] : A[i1 + (size_t)lda * q];
    const double b0 = Bm[q + (size_t)ldb * j0], b1 = Bm[q + (size_t)ldb * j1];
    acc[0][0] += a0 * b0; acc[0][1] += a0 * b1;
    acc[1][0] += a1 * b0; acc[1][1] += a1 * b1;
  }
}

// C (m x n) = epi(i, j, sum_k op(A)(i, k) B(k, j)).  Each thread computes rows {i, i + mh} x columns {j, j + nh} (mh, nh: half of m, n
// rounded up; at an odd m or n the second row / column is the first again, computed twice and stored once), consecutive threads take
// consecutive i.
template <bool TA, class Epi>
DJ_DEV void lqr_gemm(int m, int n, int kd, const double* A, int lda, const double* Bm, int ldb, Epi epi) {
  const int mh = (m + 1) >> 1, nh = (n + 1) >> 1;
  for (int tile = threadIdx.x; tile < mh * nh; tile += blockDim.x) {
    const int i0 = tile % mh, j0 = tile / mh;
    const int i1 = i0 + mh < m ? i0 + mh : i0, j1 = j0 + nh < n ? j0 + nh : j0;
    double acc[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
    lqr_tile<TA>(acc, A, lda, Bm, ldb, i0, i1, j0, j1, kd);
    epi(i0, j0, acc[0][0]);
    if (j1 != j0) epi(i0, j1, acc[0][1]);
    if (i1 != i0) {
      epi(i1, j0, acc[1][0]);
      if (j1 != j0) epi(i1, j1, acc[1][1]);
    }
  }
}

__global__ void __launch_bounds__(DJ_LQR_MAX_THREADS, 1) dojo_lqr_backward_kernel(const LqrArgs a) {
  extern __shared__ double lqr_arena[];
  const int e = blockIdx.x, tid = threadIdx.x, nth = blockDim.x;
  const int nu = a.nu, nx = 2 * nu, na = a.na, B = a.B;
  const int lx = nx + 1, ln = lqr_odd(na);
  const size_t xx = (size_t)nx * nx, xu = (size_t)nx * nu;
  double* S1 = lqr_arena;                  // P -> Qxx -> the next P (in place)  [lx x nx]
  double* S2 = S1 + (size_t)lx * nx;       // A -> Cholesky factor L [ln x na], then W = Quu_aa Y - Qa [ln x nx] behind it
  double* S3 = S2 + (size_t)lx * nx;       // PA -> Y = (Quu_aa + mu I)^-1 [Qa, -Qu_a]  [ln x (nx + 1)]
  double* Ba = S3 + (size_t)lx * nx;       // B[:, act]  [lx x na]
  double* PB = Ba + (size_t)lx * nu;       // P B[:, act]  [lx x na]
  double* Qa = PB + (size_t)lx * nu;       // Qux[act, :]  [ln x nx]
  double* Quu = Qa + (size_t)(nu + 1) * nx;  // Quu[act, act] without mu  [ln x na]
  double* p = Quu + (size_t)(nu + 1) * nu;   // [nx]
  double* dx = p + nx;           // x_bar_t - xg_t  [nx]
  double* Qx = dx + nx;          // [nx]
  double* du = Qx + nx;          // u_bar_t - ug_t  [nu]
  double* Qu = du + nu;          // Qu[act], then Quu_aa k + Qu_a  [na]
  double* flag = Qu + nu;        // [0]: the Cholesky failed
  int* act = (int*)(flag + 2);   // [na] active input indices
  for (int i = tid; i < na; i += nth) act[i] = a.act[i];
  const double mu = a.mu ? a.mu[e] : 0.0;
  const size_t ce_f = a.envs > 1 ? e : 0;
  const double* Qf = a.Qf + ce_f * xx;
  double dV1 = 0.0, dV2 = 0.0;  // thread 0's running sums
  int fail = 0;

  // P_T = Q_f, p_T = Q_f (x_T - xg_T)
  {
    const double* x = a.X + ((size_t)a.T * B + e) * nx;
    const double* g = a.xgf ? a.xgf + ce_f * nx : nullptr;
    for (int i = tid; i < nx; i += nth) dx[i] = g ? x[i] - g[i] : x[i];
    for (size_t i = tid; i < xx; i += nth) S1[i % nx + (size_t)lx * (i / nx)] = Qf[i];
    __syncthreads();
    for (int i = tid; i < nx; i += nth) {
      double s = 0.0;
      for (int j = 0; j < nx; ++j) s += Qf[i + (size_t)nx * j] * dx[j];
      p[i] = s;
    }
  }

  int t = a.T - 1;
  for (; t >= 0; --t) {
    const size_t pr = (size_t)t * B + e;                                           // pair (t, e)
    const size_t ce = (size_t)(a.steps > 1 ? t : 0) * a.envs + (a.envs > 1 ? e : 0);  // cost entry (t, e)
    const double* Q = a.Q + ce * xx;
    const double* R = a.R + ce * nu * nu;
    const double* Gx = a.Gx + pr * xx;
    const double* Gu = a.Gu + pr * xu;
    __syncthreads();  // the previous step's P and p are complete
    // (a) A_t, the active columns of B_t, dx, du
    for (size_t i = tid; i < xx; i += nth) S2[i % nx + (size_t)lx * (i / nx)] = Gx[i];
    for (size_t i = tid; i < (size_t)nx * na; i += nth) Ba[i % nx + (size_t)lx * (i / nx)] = Gu[(i % nx) + (size_t)nx * act[i / nx]];
    {
      const double* x = a.X + pr * nx;
      const double* g = a.xg ? a.xg + ce * nx : nullptr;
      for (int i = tid; i < nx; i += nth) dx[i] = g ? x[i] - g[i] : x[i];
      const double* u = a.U ? a.U + pr * nu : nullptr;
      const double* gu = a.ug ? a.ug + ce * nu : nullptr;
      for (int i = tid; i < nu; i += nth) du[i] = (u ? u[i] : 0.0) - (gu ? gu[i] : 0.0);
    }
    __syncthreads();
    // (b) PA = P A, PB = P B_a; Qx = Q dx + A'p, Qu_a = R[act, :] du + B_a'p
    lqr_gemm<false>(nx, nx, nx, S1, lx, S2, lx, [&](int i, int j, double v) { S3[i + (size_t)lx * j] = v; });
    lqr_gemm<false>(nx, na, nx, S1, lx, Ba, lx, [&](int i, int j, double v) { PB[i + (size_t)lx * j] = v; });
    for (int i = tid; i < nx + na; i += nth) {
      double s = 0.0, r = 0.0;
      if (i < nx) {
        for (int j = 0; j < nx; ++j) s += Q[i + (size_t)nx * j] * dx[j];
        for (int j = 0; j < nx; ++j) r += S2[j + (size_t)lx * i] * p[j];
        Qx[i] = s + r;
      } else {
        const int ia = i - nx, iu = act[ia];
        for (int j = 0; j < nu; ++j) s += R[iu + (size_t)nu * j] * du[j];
        for (int j = 0; j < nx; ++j) r += Ba[j + (size_t)lx * ia] * p[j];
        Qu[ia] = s + r;
      }
    }
    __syncthreads();
    // (c) Qxx = Q + A'PA over P, Qa = B_a'PA, Quu_aa = R[act, act] + B_a'PB
    lqr_gemm<true>(nx, nx, nx, S2, lx, S3, lx, [&](int i, int j, double v) { S1[i + (size_t)lx * j] = Q[i + (size_t)nx * j] + v; });
    lqr_gemm<true>(na, nx, nx, Ba, lx, S3, lx, [&](int i, int j, double v) { Qa[i + (size_t)ln * j] = v; });
    lqr_gemm<true>(na, na, nx, Ba, lx, PB, lx,
                   [&](int i, int j, double v) { Quu[i + (size_t)ln * j] = R[act[i] + (size_t)nu * act[j]] + v; });
    __syncthreads();
    // (d) L L' = Quu_aa + mu I (right-looking, lower triangle of S2, by warp 0), and the right-hand sides [Qa, -Qu_a] into S3
    double* L = S2;
    for (int i = tid; i < na * na; i += nth) L[i % na + (size_t)ln * (i / na)] = Quu[i % na + (size_t)ln * (i / na)] + ((i % na) == (i / na) ? mu : 0.0);
    for (size_t i = tid; i < (size_t)na * (nx + 1); i += nth) {
      const size_t r = i % na, c = i / na;
      S3[r + (size_t)ln * c] = c < (size_t)nx ? Qa[r + (size_t)ln * c] : -Qu[r];
    }
    if (tid == 0) flag[0] = 0.0;
    __syncthreads();
    if (tid < 32) {
      for (int j = 0; j < na; ++j) {
        if (tid == 0) {
          const double d = L[j + (size_t)ln * j];
          if (d > 0.0 && d < INFINITY) L[j + (size_t)ln * j] = sqrt(d);
          else flag[0] = 1.0;
        }
        __syncwarp();
        if (flag[0] != 0.0) break;
        const double ljj = L[j + (size_t)ln * j];
        for (int i = j + 1 + tid; i < na; i += 32) L[i + (size_t)ln * j] /= ljj;
        __syncwarp();
        for (int r = j + 1 + tid; r < na; r += 32) {  // one lane per row of the trailing lower triangle
          const double lrj = L[r + (size_t)ln * j];
          for (int c = j + 1; c <= r; ++c) L[r + (size_t)ln * c] -= lrj * L[c + (size_t)ln * j];
        }
        __syncwarp();
      }
    }
    __syncthreads();
    if (flag[0] != 0.0) { fail = 1; break; }
    // (e) Y = L'^-1 L^-1 [Qa, -Qu_a], one column per thread
    for (int c = tid; c <= nx; c += nth) {
      double* y = S3 + (size_t)ln * c;
      for (int i = 0; i < na; ++i) {
        double s = y[i];
        for (int q = 0; q < i; ++q) s -= L[i + (size_t)ln * q] * y[q];
        y[i] = s / L[i + (size_t)ln * i];
      }
      for (int i = na - 1; i >= 0; --i) {
        double s = y[i];
        for (int q = i + 1; q < na; ++q) s -= L[q + (size_t)ln * i] * y[q];
        y[i] = s / L[i + (size_t)ln * i];
      }
    }
    __syncthreads();
    // (f) outputs K_t, k_t; W = Quu_aa Y_K - Qa behind L; Qu <- Quu_aa k + Qu_a; dV
    const double* Y = S3;
    const double* kk = S3 + (size_t)ln * nx;
    double* W = S2 + (size_t)ln * na;
    {
      double* Ko = a.K + pr * nu * nx;
      double* ko = a.k + pr * nu;
      for (size_t i = tid; i < xu; i += nth) Ko[i] = 0.0;
      for (int i = tid; i < nu; i += nth) ko[i] = 0.0;
      __syncthreads();  // the zeros land before the active rows (one thread may write both)
      for (size_t i = tid; i < (size_t)na * nx; i += nth) Ko[act[i % na] + (size_t)nu * (i / na)] = Y[i % na + (size_t)ln * (i / na)];
      for (int i = tid; i < na; i += nth) ko[act[i]] = kk[i];
    }
    lqr_gemm<false>(na, nx, na, Quu, ln, Y, ln, [&](int i, int j, double v) { W[i + (size_t)ln * j] = v - Qa[i + (size_t)ln * j]; });
    if (tid == 0) {
      double s1 = 0.0, s2 = 0.0;
      for (int i = 0; i < na; ++i) {
        double qk = 0.0;
        for (int j = 0; j < na; ++j) qk += Quu[i + (size_t)ln * j] * kk[j];
        s1 += kk[i] * Qu[i];
        s2 += kk[i] * qk;
        Qu[i] += qk;
      }
      dV1 += s1; dV2 += 0.5 * s2;
    }
    __syncthreads();
    // (g) P = Qxx + Y_K'W - Qa'Y_K (in place over Qxx), p = Qx - Y_K'(Quu k + Qu) + Qa'k
    lqr_gemm<true>(nx, nx, na, Y, ln, W, ln, [&](int i, int j, double v) { S1[i + (size_t)lx * j] += v; });
    __syncthreads();
    lqr_gemm<true>(nx, nx, na, Qa, ln, Y, ln, [&](int i, int j, double v) { S1[i + (size_t)lx * j] -= v; });
    for (int i = tid; i < nx; i += nth) {
      double s = Qx[i];
      for (int j = 0; j < na; ++j) s += Qa[j + (size_t)ln * i] * kk[j] - Y[j + (size_t)ln * i] * Qu[j];
      p[i] = s;
    }
    __syncthreads();
    for (int q = tid; q < nx * nx; q += nth) {  // symmetrise: one thread per pair r < c
      const int r = q % nx, c = q / nx;
      if (r < c) {
        const double v = 0.5 * (S1[r + (size_t)lx * c] + S1[c + (size_t)lx * r]);
        S1[r + (size_t)lx * c] = v;
        S1[c + (size_t)lx * r] = v;
      }
    }
  }
  if (fail) {  // the Cholesky failed at step t: K_s, k_s for s <= t and dV are NaN
    const double nan = NAN;
    for (int s = 0; s <= t; ++s) {
      const size_t pr = (size_t)s * B + e;
      for (size_t i = tid; i < xu; i += nth) a.K[pr * xu + i] = nan;
      for (int i = tid; i < nu; i += nth) a.k[pr * nu + i] = nan;
    }
  }
  if (tid == 0) {
    if (a.dV) { a.dV[2 * (size_t)e] = fail ? NAN : dV1; a.dV[2 * (size_t)e + 1] = fail ? NAN : dV2; }
    if (a.status) a.status[e] = fail ? t + 1 : 0;
  }
}

}  // namespace dj
