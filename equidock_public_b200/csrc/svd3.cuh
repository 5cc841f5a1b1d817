// 3x3 Jacobi SVD and fp64 warp reductions shared by the docking head (head.cu), the RMSD meter and the graph builder
// (graph_build.cu).
#pragma once

namespace eqd {

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// 3x3 SVD A = U diag(S) V^T by one-sided (Hestenes) Jacobi in fp64, singular values sorted
// descending.  U is orthonormal for every input: columns of U that belong to a singular value at
// rounding level of S[0] are completed from V (see the end).
__device__ inline void svd3(const double (&A)[9], double (&U)[9], double (&S)[3], double (&V)[9]) {
  double G[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) G[q] = A[q];
  V[0] = 1; V[1] = 0; V[2] = 0; V[3] = 0; V[4] = 1; V[5] = 0; V[6] = 0; V[7] = 0; V[8] = 1;
  for (int sweep = 0; sweep < 40; ++sweep) {
    double off = 0.0;
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      double alpha = 0, beta = 0, gamma = 0;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        alpha += G[r * 3 + p] * G[r * 3 + p];
        beta += G[r * 3 + q] * G[r * 3 + q];
        gamma += G[r * 3 + p] * G[r * 3 + q];
      }
      if (gamma == 0.0) continue;
      double lim = sqrt(alpha * beta);
      if (fabs(gamma) <= 1e-18 * lim) continue;
      off = fmax(off, fabs(gamma) / fmax(lim, 1e-300));
      double zeta = (beta - alpha) / (2.0 * gamma);
      // |zeta| > 1e153 (a column at rounding level of the other): zeta * zeta overflows from ~1.3e154 on and the textbook t
      // would be 0, which stalls the sweep; t = 1 / (2 zeta) is its limit there
      double t = fabs(zeta) > 1e153 ? 0.5 / zeta : (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
      double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        double gp = G[r * 3 + p], gq = G[r * 3 + q];
        G[r * 3 + p] = c * gp - sn * gq;
        G[r * 3 + q] = sn * gp + c * gq;
        double vp = V[r * 3 + p], vq = V[r * 3 + q];
        V[r * 3 + p] = c * vp - sn * vq;
        V[r * 3 + q] = sn * vp + c * vq;
      }
    }
    if (off < 1e-15) break;
  }
  double nrm[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) nrm[c] = sqrt(G[c] * G[c] + G[3 + c] * G[3 + c] + G[6 + c] * G[6 + c]);
  // sort columns by descending singular value (3-element network)
  int idx[3] = {0, 1, 2};
#define EQD_CSWAP(a, b) if (nrm[idx[a]] < nrm[idx[b]]) { int t_ = idx[a]; idx[a] = idx[b]; idx[b] = t_; }
  EQD_CSWAP(0, 1) EQD_CSWAP(1, 2) EQD_CSWAP(0, 1)
#undef EQD_CSWAP
  double Vs[9];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    int sc = idx[c];
    S[c] = nrm[sc];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      Vs[r * 3 + c] = V[r * 3 + sc];
      U[r * 3 + c] = nrm[sc] > 0.0 ? G[r * 3 + sc] / nrm[sc] : 0.0;
    }
  }
#pragma unroll
  for (int q = 0; q < 9; ++q) V[q] = Vs[q];
  // Rank-deficient A (collinear or coplanar point sets, 1-3 points): a column whose singular value is at rounding level of
  // S[0] carries no direction -- its normalised G column is zero or noise.  Complete U from the matching columns of V,
  // Gram-Schmidt against the columns already fixed, so that U stays orthonormal: a symmetric PSD A (Kabsch of a trace onto
  // itself) then gives U = V, i.e. R = I, and any other A an optimal proper rotation after the reflection fix.
  const double tol = 64.0 * 2.220446049250313e-16 * S[0];
  if (!(S[0] > tol)) {            // A = 0
    U[0] = V[0]; U[3] = V[3]; U[6] = V[6];
  }
  if (!(S[1] > tol)) {            // rank <= 1: v1, else v2, minus its u0 component (one of the two keeps |w|^2 >= 1/2)
    double w[3], ww = 0.0;
    for (int k = 1; k < 3 && ww < 0.5; ++k) {
      const double d = U[0] * V[k] + U[3] * V[3 + k] + U[6] * V[6 + k];
      ww = 0.0;
      for (int r = 0; r < 3; ++r) {
        w[r] = V[r * 3 + k] - d * U[r * 3];
        ww += w[r] * w[r];
      }
    }
    const double inv = 1.0 / sqrt(ww);
    for (int r = 0; r < 3; ++r) U[r * 3 + 1] = w[r] * inv;
  }
  if (!(S[2] > tol)) {            // rank <= 2: u2 = +-(u0 x u1), the sign of v2
    const double w[3] = {U[3] * U[7] - U[6] * U[4], U[6] * U[1] - U[0] * U[7], U[0] * U[4] - U[3] * U[1]};
    const double sg = w[0] * V[2] + w[1] * V[5] + w[2] * V[8] < 0.0 ? -1.0 : 1.0;
    for (int r = 0; r < 3; ++r) U[r * 3 + 2] = sg * w[r];
  }
}


}  // namespace eqd
