// The cyclic Jacobi eigen-solve of a symmetric R x R matrix, shared by CPD-ALS (cpd.cu: the
// pseudo-inverse fallback of the normal equations) and Tucker (tucker.cu: the Rayleigh-Ritz step).
// Included inside the includer's anonymous namespace.
#pragma once

// Pseudo-inverse P of the symmetric R x R matrix A (overwritten) by a Jacobi eigen-solve, with
// the LAPACK default cut-off (rcond < 0 -> machine eps); V: R x R scratch.  Returns the
// effective rank.  Runs on the host (pinv_solve_rows) and in one thread of k_form_chol.  On return
// A holds the eigenvalues on its diagonal (A[e + e * R]) and V the eigenvectors as the columns of
// a row-major matrix (V[e + i * R] is component i of eigenvector e).
__host__ __device__ int jacobi_pinv(double * A, double * V, int R, double * P) {
  for (int x = 0; x < R * R; ++x) V[x] = 0.0;
  for (int i = 0; i < R; ++i) V[i + i * R] = 1.0;
  for (int sweep = 0; sweep < 64; ++sweep) {
    double off = 0;
    for (int p = 0; p < R; ++p)
      for (int q = p + 1; q < R; ++q) off += A[q + p * R] * A[q + p * R];
    if (off < 1e-300) break;
    for (int p = 0; p < R; ++p)
      for (int q = p + 1; q < R; ++q) {
        const double apq = A[q + p * R];
        if (fabs(apq) < 1e-300) continue;
        const double theta = (A[q + q * R] - A[p + p * R]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < R; ++k) {
          const double akp = A[p + k * R], akq = A[q + k * R];
          A[p + k * R] = c * akp - s * akq;
          A[q + k * R] = s * akp + c * akq;
        }
        for (int k = 0; k < R; ++k) {
          const double apk = A[k + p * R], aqk = A[k + q * R];
          A[k + p * R] = c * apk - s * aqk;
          A[k + q * R] = s * apk + c * aqk;
        }
        for (int k = 0; k < R; ++k) {
          const double vkp = V[p + k * R], vkq = V[q + k * R];
          V[p + k * R] = c * vkp - s * vkq;
          V[q + k * R] = s * vkp + c * vkq;
        }
      }
  }
  double dmax = 0;
  for (int i = 0; i < R; ++i) dmax = fmax(dmax, fabs(A[i + i * R]));
  const double cut = dmax * 2.220446049250313e-16;
  for (int x = 0; x < R * R; ++x) P[x] = 0.0;
  int erank = 0;
  for (int e = 0; e < R; ++e) {
    const double d = A[e + e * R];
    if (fabs(d) <= cut) continue;
    ++erank;
    for (int i = 0; i < R; ++i)
      for (int j = 0; j < R; ++j) P[j + i * R] += V[e + i * R] * V[e + j * R] / d;
  }
  return erank;
}
