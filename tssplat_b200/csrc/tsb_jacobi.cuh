// Cyclic Jacobi rotation of a symmetric 3x3 matrix in fp64 registers, shared by the preconditioner blocks (tsb_solver.cu)
// and the projected Hessian (tsb_psd.cu).
#pragma once

namespace tsb {

// One Jacobi rotation of a symmetric 3x3 matrix that zeroes a_pq; r is the third index, (v?p, v?q) are columns p and q
// of the eigenvector matrix.
__device__ __forceinline__ void jacobi_rot(double &app, double &aqq, double &apq, double &apr, double &aqr, double &v0p,
                                           double &v0q, double &v1p, double &v1q, double &v2p, double &v2q) {
  if (apq == 0.0) return;
  const double theta = (aqq - app) / (2.0 * apq);
  const double t = copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
  const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
  app -= t * apq; aqq += t * apq; apq = 0.0;
  double a = c * apr - s * aqr; aqr = s * apr + c * aqr; apr = a;
  a = c * v0p - s * v0q; v0q = s * v0p + c * v0q; v0p = a;
  a = c * v1p - s * v1q; v1q = s * v1p + c * v1q; v1p = a;
  a = c * v2p - s * v2q; v2q = s * v2p + c * v2q; v2p = a;
}

constexpr int kJacobiSweeps = 8;

}  // namespace tsb
