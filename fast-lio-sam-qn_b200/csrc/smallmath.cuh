// smallmath.cuh -- tiny fp64 device helpers shared by gicp.cu, knn_large.cu and quatro.cu.
#pragma once
#include <cuda_runtime.h>

namespace b200 {

// Full eigen-decomposition of a symmetric 3x3 by cyclic Jacobi (fp64): eigenvalues in w (unsorted), eigenvectors in
// the columns of V.  The non-default regularisation methods and sym3_smallest_evec's near-degenerate case need it (cold
// paths).
static __device__ __noinline__ void sym3_eigen_jacobi(const double a[6], double w[3], double V[3][3]) {
  double A[3][3] = {{a[0], a[1], a[2]}, {a[1], a[3], a[4]}, {a[2], a[4], a[5]}};
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) V[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 16; sweep++) {
    const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
    const double dg = A[0][0] * A[0][0] + A[1][1] * A[1][1] + A[2][2] * A[2][2];
    if (off == 0.0 || off <= 1e-34 * dg) break;
    for (int pq = 0; pq < 3; pq++) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2, r = 3 - p - q;
      const double apq = A[p][q];
      if (apq == 0.0) continue;
      const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
      const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
      const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
      A[p][p] -= t * apq;
      A[q][q] += t * apq;
      A[p][q] = A[q][p] = 0.0;
      const double arp = A[r][p], arq = A[r][q];
      A[r][p] = A[p][r] = c * arp - s * arq;
      A[r][q] = A[q][r] = s * arp + c * arq;
      for (int k = 0; k < 3; k++) {
        const double vp = V[k][p], vq = V[k][q];
        V[k][p] = c * vp - s * vq;
        V[k][q] = s * vp + c * vq;
      }
    }
  }
  w[0] = A[0][0]; w[1] = A[1][1]; w[2] = A[2][2];
}

// Eigenvector of the smallest eigenvalue of a symmetric 3x3, fp64, non-iterative:
// eigenvalue by the trigonometric closed form on the matrix scaled to unit max entry, eigenvector as the
// best-conditioned cross product of two rows of (A - lambda I), then ONE inverse-iteration-free polish by
// re-orthogonalising against the residual.  (A cyclic-Jacobi version was measured first: its fp64 div/sqrt chains
// were ~30% of k_covariance's instructions.)  Accuracy ~1e-13 relative for the plane-like neighbourhoods GICP uses;
// when the two smallest eigenvalues coincide any vector of that eigenspace is returned, as with an SVD.
// Where the two smallest eigenvalues are g apart with g << p (the spread; near-collinear neighbourhoods: poles, edges),
// r -> 1 and acos has infinite slope there: the closed-form lambda errs by ~eps p^2 / g and the cross products turn that
// into an eigenvector error ~eps (p/g)^2, where the problem itself only allows ~eps p / g (an fp64 restatement of this
// code errs by 3e-5 rad on near-collinear points of a raw scan; one Rayleigh-quotient refinement of lambda was measured
// to leave errors of 0.4 rad on a 2e-4 m-thick edge, where lambda's error exceeds g).  So below phi = 1e-3
// (g / p ~ 3.5e-3) the vector comes from the backward-stable cyclic Jacobi instead
// (tests/test_gpu_fpfh_dense.py checks the normals against that eigen-gap bound).
__device__ __forceinline__ void sym3_smallest_evec(double a00, double a01, double a02, double a11, double a12,
                                                   double a22, double n[3]) {
  const double mx = fmax(fmax(fmax(fabs(a00), fabs(a01)), fmax(fabs(a02), fabs(a11))), fmax(fabs(a12), fabs(a22)));
  if (mx == 0.0) {
    n[0] = 0.0; n[1] = 0.0; n[2] = 1.0;
    return;
  }
  const double is = 1.0 / mx;
  a00 *= is; a01 *= is; a02 *= is; a11 *= is; a12 *= is; a22 *= is;
  const double off = a01 * a01 + a02 * a02 + a12 * a12;
  double lam;
  if (off == 0.0) {
    lam = fmin(a00, fmin(a11, a22));
  } else {
    const double q = (a00 + a11 + a22) * (1.0 / 3.0);
    const double b00 = a00 - q, b11 = a11 - q, b22 = a22 - q;
    const double p = sqrt((b00 * b00 + b11 * b11 + b22 * b22 + 2.0 * off) * (1.0 / 6.0));
    const double ip = 1.0 / p;
    const double c00 = b00 * ip, c01 = a01 * ip, c02 = a02 * ip, c11 = b11 * ip, c12 = a12 * ip, c22 = b22 * ip;
    double r = 0.5 * (c00 * (c11 * c22 - c12 * c12) - c01 * (c01 * c22 - c12 * c02) + c02 * (c01 * c12 - c11 * c02));
    r = fmin(1.0, fmax(-1.0, r));
    const double phi = acos(r) * (1.0 / 3.0);
    if (phi < 1e-3) {  // the two smallest eigenvalues nearly coincide: see above
      const double a6[6] = {a00, a01, a02, a11, a12, a22};
      double w[3], V[3][3];
      sym3_eigen_jacobi(a6, w, V);
      const int k = w[0] <= w[1] ? (w[0] <= w[2] ? 0 : 2) : (w[1] <= w[2] ? 1 : 2);
      n[0] = V[0][k]; n[1] = V[1][k]; n[2] = V[2][k];
      return;
    }
    lam = q + 2.0 * p * cos(phi + 2.0943951023931954923);  // smallest root
  }
  // rows of (A - lam I); the eigenvector is orthogonal to all three
  const double r0x = a00 - lam, r0y = a01, r0z = a02;
  const double r1x = a01, r1y = a11 - lam, r1z = a12;
  const double r2x = a02, r2y = a12, r2z = a22 - lam;
  const double c0x = r0y * r1z - r0z * r1y, c0y = r0z * r1x - r0x * r1z, c0z = r0x * r1y - r0y * r1x;
  const double c1x = r0y * r2z - r0z * r2y, c1y = r0z * r2x - r0x * r2z, c1z = r0x * r2y - r0y * r2x;
  const double c2x = r1y * r2z - r1z * r2y, c2y = r1z * r2x - r1x * r2z, c2z = r1x * r2y - r1y * r2x;
  const double d0 = c0x * c0x + c0y * c0y + c0z * c0z, d1 = c1x * c1x + c1y * c1y + c1z * c1z,
               d2 = c2x * c2x + c2y * c2y + c2z * c2z;
  double vx = c0x, vy = c0y, vz = c0z, dm = d0;
  if (d1 > dm) { vx = c1x; vy = c1y; vz = c1z; dm = d1; }
  if (d2 > dm) { vx = c2x; vy = c2y; vz = c2z; dm = d2; }
  if (dm == 0.0) {  // (A - lam I) has rank <= 1: pick any vector orthogonal to its dominant row
    double rx = r0x, ry = r0y, rz = r0z;
    double rm = r0x * r0x + r0y * r0y + r0z * r0z;
    const double m1 = r1x * r1x + r1y * r1y + r1z * r1z, m2 = r2x * r2x + r2y * r2y + r2z * r2z;
    if (m1 > rm) { rx = r1x; ry = r1y; rz = r1z; rm = m1; }
    if (m2 > rm) { rx = r2x; ry = r2y; rz = r2z; rm = m2; }
    if (rm == 0.0) { n[0] = 0.0; n[1] = 0.0; n[2] = 1.0; return; }
    if (fabs(rx) <= fabs(ry) && fabs(rx) <= fabs(rz)) { vx = 0.0; vy = -rz; vz = ry; }
    else if (fabs(ry) <= fabs(rz)) { vx = -rz; vy = 0.0; vz = rx; }
    else { vx = -ry; vy = rx; vz = 0.0; }
    dm = vx * vx + vy * vy + vz * vz;
  }
  const double inv = rsqrt(dm);
  n[0] = vx * inv; n[1] = vy * inv; n[2] = vz * inv;
}

// inverse of a symmetric 3x3 given as (xx,xy,xz,yy,yz,zz); result in the same packing
__device__ __forceinline__ void sym3_inverse(const double a[6], double o[6]) {
  double c00 = a[3] * a[5] - a[4] * a[4];
  double c01 = a[2] * a[4] - a[1] * a[5];
  double c02 = a[1] * a[4] - a[2] * a[3];
  double det = a[0] * c00 + a[1] * c01 + a[2] * c02;
  double id = 1.0 / det;
  o[0] = c00 * id;
  o[1] = c01 * id;
  o[2] = c02 * id;
  o[3] = (a[0] * a[5] - a[2] * a[2]) * id;
  o[4] = (a[1] * a[2] - a[0] * a[4]) * id;
  o[5] = (a[0] * a[3] - a[1] * a[1]) * id;
}

// RegularizationMethod (nano_gicp_impl.hpp:323-353) of the covariance (cxx, cxy, cxz, cyy, cyz, czz), stored packed at o.
// method: 0 NONE, 1 MIN_EIG, 2 NORMALIZED_MIN_EIG, 3 PLANE, 4 FROBENIUS.  The epilogue of both covariance kernels
// (k_covariance in gicp.cu, k_covariance_large in knn_large.cu).
// PLANE: for symmetric PSD input U diag(1,1,eps) V^T == I - (1-eps) n n^T with n the eigenvector of the smallest
// eigenvalue (SURVEY.md App. A.2), so only n is computed.
__device__ __forceinline__ void cov_regularize_store(double* o, double cxx, double cxy, double cxz, double cyy, double cyz,
                                                     double czz, int method) {
  if (method == 3) {  // PLANE, the default (nano_gicp_impl.hpp:61, 341-343)
    double n[3];
    sym3_smallest_evec(cxx, cxy, cxz, cyy, cyz, czz, n);
    const double w = 1.0 - 1e-3;
    o[0] = 1.0 - w * n[0] * n[0];
    o[1] = -w * n[0] * n[1];
    o[2] = -w * n[0] * n[2];
    o[3] = 1.0 - w * n[1] * n[1];
    o[4] = -w * n[1] * n[2];
    o[5] = 1.0 - w * n[2] * n[2];
    return;
  }
  // cold path: the other RegularizationMethods (nano_gicp_impl.hpp:323-353)
  if (method == 0) {  // NONE
    o[0] = cxx; o[1] = cxy; o[2] = cxz; o[3] = cyy; o[4] = cyz; o[5] = czz;
  } else if (method == 4) {  // FROBENIUS: ((C + 1e-3 I)^-1 / ||.||_F)^-1 = ||(C + 1e-3 I)^-1||_F (C + 1e-3 I)
    const double cl[6] = {cxx + 1e-3, cxy, cxz, cyy + 1e-3, cyz, czz + 1e-3};
    double ci[6];
    sym3_inverse(cl, ci);
    const double nrm = sqrt(ci[0] * ci[0] + ci[3] * ci[3] + ci[5] * ci[5] + 2.0 * (ci[1] * ci[1] + ci[2] * ci[2] + ci[4] * ci[4]));
#pragma unroll
    for (int a = 0; a < 6; a++) o[a] = nrm * cl[a];
  } else {  // MIN_EIG / NORMALIZED_MIN_EIG: sum_i max(f(s_i), 1e-3) u_i u_i^T
    const double a6[6] = {cxx, cxy, cxz, cyy, cyz, czz};
    double wv[3], V[3][3];
    sym3_eigen_jacobi(a6, wv, V);
    double vals[3];
    const double mx = fmax(wv[0], fmax(wv[1], wv[2]));
    for (int a = 0; a < 3; a++) {
      const double sgl = fmax(wv[a], 0.0);  // singular value of a PSD matrix
      const double f = method == 2 ? sgl / mx : sgl;
      // std::max(f, 1e-3) as the reference's (s / s.maxCoeff()).array().max(1e-3): at a zero covariance (k = 1, or k copies
      // of one point) NORMALIZED_MIN_EIG gives 0 / 0 and the NaN is kept (fmax would return 1e-3)
      vals[a] = f < 1e-3 ? 1e-3 : f;
    }
    double r[6] = {0, 0, 0, 0, 0, 0};
    for (int a = 0; a < 3; a++) {
      r[0] += vals[a] * V[0][a] * V[0][a];
      r[1] += vals[a] * V[0][a] * V[1][a];
      r[2] += vals[a] * V[0][a] * V[2][a];
      r[3] += vals[a] * V[1][a] * V[1][a];
      r[4] += vals[a] * V[1][a] * V[2][a];
      r[5] += vals[a] * V[2][a] * V[2][a];
    }
#pragma unroll
    for (int a = 0; a < 6; a++) o[a] = r[a];
  }
}

}  // namespace b200
