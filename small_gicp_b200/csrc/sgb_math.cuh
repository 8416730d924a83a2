// SPDX-License-Identifier: MIT
// Per-point arithmetic of the hot path: the factor algebra of ICP / point-to-plane / GICP (+ robust kernels), the GICP
// precision matrix, the mapping of the 28 compact sums to H | b | e, and the 3x3 eigenvector of feature estimation.  No memory access pattern, no warp primitive:
// everything here is plain C++ on scalars (device functions under nvcc, plain inline functions under g++), so the SAME source that the kernels inline is also compiled
// by g++ into tests/host_math/libsgb_host_math.so and checked against the oracle and the numpy leg without a GPU
// (tests/test_device_math_on_host.py).  That library is test infrastructure; the product never loads it.
#pragma once
#include <stdint.h>
#include <vector_types.h>  // float4

#if defined(__CUDACC__)
#define SGB_HD __device__ __forceinline__
#define SGB_HHD __host__ __device__ inline  // also called by the host code of the library (sgb_capi_batch.cu)
#else
#include <cmath>
#define SGB_HD inline
#define SGB_HHD inline
#endif

namespace sgb {

constexpr int kAcc = 28;  // 6 (H_rr sym) + 9 (H_rt) + 6 (H_tt sym) + 6 (b) + 1 (e)

/// Symmetric 3x3 stored as (xx, xy, xz, yy, yz, zz).
struct Sym3 {
  double xx, xy, xz, yy, yz, zz;
};

SGB_HD Sym3 sym3_inverse(const Sym3& a) {
  // cofactors / determinant (the closed form Eigen uses for 3x3, gicp_factor.hpp:60)
  const double c00 = a.yy * a.zz - a.yz * a.yz;
  const double c01 = a.xz * a.yz - a.xy * a.zz;
  const double c02 = a.xy * a.yz - a.xz * a.yy;
  const double c11 = a.xx * a.zz - a.xz * a.xz;
  const double c12 = a.xy * a.xz - a.xx * a.yz;
  const double c22 = a.xx * a.yy - a.xy * a.xy;
  const double det = a.xx * c00 + a.xy * c01 + a.xz * c02;
  const double inv = 1.0 / det;
  return Sym3{c00 * inv, c01 * inv, c02 * inv, c11 * inv, c12 * inv, c22 * inv};
}

/// RCR = Ct + R Cs R^T (3x3 blocks of gicp_factor.hpp:59) ; returns its inverse (the fused precision matrix).
SGB_HD Sym3 gicp_precision(const double* R, const float4& sA, const float4& sB, const float4& tA, const float4& tB) {
  const double sxx = sA.x, sxy = sA.y, sxz = sA.z, syy = sA.w, syz = sB.x, szz = sB.y;
  // A = R * Cs
  double A[9];
#pragma unroll
  for (int i = 0; i < 3; i++) {
    const double r0 = R[i * 3 + 0], r1 = R[i * 3 + 1], r2 = R[i * 3 + 2];
    A[i * 3 + 0] = r0 * sxx + r1 * sxy + r2 * sxz;
    A[i * 3 + 1] = r0 * sxy + r1 * syy + r2 * syz;
    A[i * 3 + 2] = r0 * sxz + r1 * syz + r2 * szz;
  }
  Sym3 rcr;
  rcr.xx = static_cast<double>(tA.x) + (A[0] * R[0] + A[1] * R[1] + A[2] * R[2]);
  rcr.xy = static_cast<double>(tA.y) + (A[0] * R[3] + A[1] * R[4] + A[2] * R[5]);
  rcr.xz = static_cast<double>(tA.z) + (A[0] * R[6] + A[1] * R[7] + A[2] * R[8]);
  rcr.yy = static_cast<double>(tA.w) + (A[3] * R[3] + A[4] * R[4] + A[5] * R[5]);
  rcr.yz = static_cast<double>(tB.x) + (A[3] * R[6] + A[4] * R[7] + A[5] * R[8]);
  rcr.zz = static_cast<double>(tB.y) + (A[6] * R[6] + A[7] * R[7] + A[8] * R[8]);
  return sym3_inverse(rcr);
}

/// Accumulate one point's  J^T M J | J^T M r | 1/2 r^T M r  (scaled by w) into acc[28], where
/// J = [R skew(p) | -R]  (icp_factor.hpp:45-47) and M is the 3x3 weight in the target frame:
/// identity (ICP), diag(n.^2) (point-to-plane, plane_icp_factor.hpp:46-55) or (Ct + R Cs R^T)^-1 (GICP).
/// Returns the unweighted error e.
template <int ROBUST>
SGB_HD void accumulate_factor(const double* R, const Sym3& M, double rx, double ry, double rz, double px, double py, double pz,
                                                  double robust_c, double* acc) {
  // Mr, e
  const double mrx = M.xx * rx + M.xy * ry + M.xz * rz;
  const double mry = M.xy * rx + M.yy * ry + M.yz * rz;
  const double mrz = M.xz * rx + M.yz * ry + M.zz * rz;
  const double e = 0.5 * (rx * mrx + ry * mry + rz * mrz);
  double w = 1.0;
  if (ROBUST == 1) {  // Huber, robust_kernel.hpp:24-27 on sqrt(e) (robust_kernel.hpp:84)
    const double x = sqrt(e);
    w = x < robust_c ? 1.0 : robust_c / x;
  } else if (ROBUST == 2) {  // Cauchy, robust_kernel.hpp:47 : c / (c + x^2) with x = sqrt(e)
    const double x = sqrt(e);
    w = robust_c / (robust_c + x * x);
  }
  // MR = M * R ; D = R^T * MR (symmetric)
  double MR[9];
#pragma unroll
  for (int j = 0; j < 3; j++) {
    const double r0 = R[0 + j], r1 = R[3 + j], r2 = R[6 + j];
    MR[0 + j] = M.xx * r0 + M.xy * r1 + M.xz * r2;
    MR[3 + j] = M.xy * r0 + M.yy * r1 + M.yz * r2;
    MR[6 + j] = M.xz * r0 + M.yz * r1 + M.zz * r2;
  }
  const double d00 = w * (R[0] * MR[0] + R[3] * MR[3] + R[6] * MR[6]);
  const double d01 = w * (R[0] * MR[1] + R[3] * MR[4] + R[6] * MR[7]);
  const double d02 = w * (R[0] * MR[2] + R[3] * MR[5] + R[6] * MR[8]);
  const double d11 = w * (R[1] * MR[1] + R[4] * MR[4] + R[7] * MR[7]);
  const double d12 = w * (R[1] * MR[2] + R[4] * MR[5] + R[7] * MR[8]);
  const double d22 = w * (R[2] * MR[2] + R[5] * MR[5] + R[8] * MR[8]);
  // g = w * R^T (M r)
  const double gx = w * (R[0] * mrx + R[3] * mry + R[6] * mrz);
  const double gy = w * (R[1] * mrx + R[4] * mry + R[7] * mrz);
  const double gz = w * (R[2] * mrx + R[5] * mry + R[8] * mrz);
  // U = skew(p) * D : column j = p x D[:, j]      (H_rt = U)
  const double u00 = py * d02 - pz * d01, u01 = py * d12 - pz * d11, u02 = py * d22 - pz * d12;
  const double u10 = pz * d00 - px * d02, u11 = pz * d01 - px * d12, u12 = pz * d02 - px * d22;
  const double u20 = px * d01 - py * d00, u21 = px * d11 - py * d01, u22 = px * d12 - py * d02;
  // H_rr = skew(p)^T D skew(p) : row i = p x U[i, :]
  acc[0] += py * u02 - pz * u01;
  acc[1] += pz * u00 - px * u02;
  acc[2] += px * u01 - py * u00;
  acc[3] += pz * u10 - px * u12;
  acc[4] += px * u11 - py * u10;
  acc[5] += px * u21 - py * u20;
  acc[6] += u00;
  acc[7] += u01;
  acc[8] += u02;
  acc[9] += u10;
  acc[10] += u11;
  acc[11] += u12;
  acc[12] += u20;
  acc[13] += u21;
  acc[14] += u22;
  acc[15] += d00;
  acc[16] += d01;
  acc[17] += d02;
  acc[18] += d11;
  acc[19] += d12;
  acc[20] += d22;
  // b = J^T M r = [ g x p ; -g ]
  acc[21] += gy * pz - gz * py;
  acc[22] += gz * px - gx * pz;
  acc[23] += gx * py - gy * px;
  acc[24] -= gx;
  acc[25] -= gy;
  acc[26] -= gz;
  acc[27] += w * e;
}

/// GICP weight in the SOURCE frame.  With R orthogonal,  R^T (Ct + R Cs R^T)^-1 R = (R^T Ct R + Cs)^-1 =: D.  D is all the
/// Hessian blocks need (H_tt = D, H_rt = skew(p) D, H_rr = skew(p)^T D skew(p)), and  R^T M r = D (R^T r),
/// r^T M r = (R^T r)^T D (R^T r):  the target-frame precision matrix M of gicp_factor.hpp:59-60 never has to be formed
/// (~50 of the ~240 FP64 operations per point of the target-frame formulation above; same value up to rounding).
SGB_HD Sym3 gicp_precision_source(const double* R, const float4& sA, const float4& sB, const float4& tA, const float4& tB) {
  const double txx = tA.x, txy = tA.y, txz = tA.z, tyy = tA.w, tyz = tB.x, tzz = tB.y;
  double B[9];  // B = Ct * R
#pragma unroll
  for (int j = 0; j < 3; j++) {
    const double r0 = R[0 + j], r1 = R[3 + j], r2 = R[6 + j];
    B[0 + j] = txx * r0 + txy * r1 + txz * r2;
    B[3 + j] = txy * r0 + tyy * r1 + tyz * r2;
    B[6 + j] = txz * r0 + tyz * r1 + tzz * r2;
  }
  Sym3 n;  // N = Cs + R^T B
  n.xx = static_cast<double>(sA.x) + (R[0] * B[0] + R[3] * B[3] + R[6] * B[6]);
  n.xy = static_cast<double>(sA.y) + (R[0] * B[1] + R[3] * B[4] + R[6] * B[7]);
  n.xz = static_cast<double>(sA.z) + (R[0] * B[2] + R[3] * B[5] + R[6] * B[8]);
  n.yy = static_cast<double>(sA.w) + (R[1] * B[1] + R[4] * B[4] + R[7] * B[7]);
  n.yz = static_cast<double>(sB.x) + (R[1] * B[2] + R[4] * B[5] + R[7] * B[8]);
  n.zz = static_cast<double>(sB.y) + (R[2] * B[2] + R[5] * B[5] + R[8] * B[8]);
  return sym3_inverse(n);
}

/// Point-to-plane weight diag(n.^2) (plane_icp_factor.hpp:46-55) carried to the source frame: D = R^T diag(n.^2) R.
SGB_HD Sym3 plane_weight_source(const double* R, double nx, double ny, double nz) {
  const double a = nx * nx, b = ny * ny, c = nz * nz;
  Sym3 d;
  d.xx = a * R[0] * R[0] + b * R[3] * R[3] + c * R[6] * R[6];
  d.xy = a * R[0] * R[1] + b * R[3] * R[4] + c * R[6] * R[7];
  d.xz = a * R[0] * R[2] + b * R[3] * R[5] + c * R[6] * R[8];
  d.yy = a * R[1] * R[1] + b * R[4] * R[4] + c * R[7] * R[7];
  d.yz = a * R[1] * R[2] + b * R[4] * R[5] + c * R[7] * R[8];
  d.zz = a * R[2] * R[2] + b * R[5] * R[5] + c * R[8] * R[8];
  return d;
}

/// One point's terms of the same sums as accumulate_factor (sum k gets t[k]), from the source-frame weight D = R^T M R and the
/// source-frame residual rs = R^T r.
template <int ROBUST>
SGB_HD void factor_terms_source(const Sym3& D, double rsx, double rsy, double rsz, double px, double py, double pz, double robust_c, double* t) {
  const double mrx = D.xx * rsx + D.xy * rsy + D.xz * rsz;
  const double mry = D.xy * rsx + D.yy * rsy + D.yz * rsz;
  const double mrz = D.xz * rsx + D.yz * rsy + D.zz * rsz;
  const double e = 0.5 * (rsx * mrx + rsy * mry + rsz * mrz);
  double w = 1.0;
  if (ROBUST == 1) {  // Huber, robust_kernel.hpp:24-27 on sqrt(e) (robust_kernel.hpp:84)
    const double x = sqrt(e);
    w = x < robust_c ? 1.0 : robust_c / x;
  } else if (ROBUST == 2) {  // Cauchy, robust_kernel.hpp:47 : c / (c + x^2) with x = sqrt(e)
    const double x = sqrt(e);
    w = robust_c / (robust_c + x * x);
  }
  const double d00 = w * D.xx, d01 = w * D.xy, d02 = w * D.xz, d11 = w * D.yy, d12 = w * D.yz, d22 = w * D.zz;
  const double gx = w * mrx, gy = w * mry, gz = w * mrz;  // g = w R^T M r
  const double u00 = py * d02 - pz * d01, u01 = py * d12 - pz * d11, u02 = py * d22 - pz * d12;
  const double u10 = pz * d00 - px * d02, u11 = pz * d01 - px * d12, u12 = pz * d02 - px * d22;
  const double u20 = px * d01 - py * d00, u21 = px * d11 - py * d01, u22 = px * d12 - py * d02;
  t[0] = py * u02 - pz * u01;
  t[1] = pz * u00 - px * u02;
  t[2] = px * u01 - py * u00;
  t[3] = pz * u10 - px * u12;
  t[4] = px * u11 - py * u10;
  t[5] = px * u21 - py * u20;
  t[6] = u00;
  t[7] = u01;
  t[8] = u02;
  t[9] = u10;
  t[10] = u11;
  t[11] = u12;
  t[12] = u20;
  t[13] = u21;
  t[14] = u22;
  t[15] = d00;
  t[16] = d01;
  t[17] = d02;
  t[18] = d11;
  t[19] = d12;
  t[20] = d22;
  t[21] = gy * pz - gz * py;
  t[22] = gz * px - gx * pz;
  t[23] = gx * py - gy * px;
  t[24] = -gx;
  t[25] = -gy;
  t[26] = -gz;
  t[27] = w * e;
}

/// Same sums as accumulate_factor, from the source-frame weight D = R^T M R and the source-frame residual rs = R^T r.
template <int ROBUST>
SGB_HD void accumulate_factor_source(const Sym3& D, double rsx, double rsy, double rsz, double px, double py, double pz, double robust_c,
                                                         double* acc) {
  double t[kAcc];
  factor_terms_source<ROBUST>(D, rsx, rsy, rsz, px, py, pz, robust_c, t);
#pragma unroll
  for (int k = 0; k < kAcc; k++) acc[k] += t[k];
}

/// The part of point_linearize_source (below, same arguments) before the sums: false if rejected (D, rs, p untouched), else the
/// source-frame weight D, the source-frame residual rs and the source point p (absolute, FP64) that factor_terms_source takes.
template <int FACTOR>
SGB_HD bool point_weight_source(const double* R, double tpx, double tpy, double tpz, double csx, double csy, double csz, double max_dist_sq_d,
                                const float4& sp, const float4* sA, const float4* sB, const float4& tq, const float4* t1, const float4* t2, Sym3& D,
                                double* rs, double* p) {
  const double sx = sp.x, sy = sp.y, sz = sp.z;
  const double qx = R[0] * sx + R[1] * sy + R[2] * sz + tpx;
  const double qy = R[3] * sx + R[4] * sy + R[5] * sz + tpy;
  const double qz = R[6] * sx + R[7] * sy + R[8] * sz + tpz;
  const double rx = static_cast<double>(tq.x) - qx, ry = static_cast<double>(tq.y) - qy, rz = static_cast<double>(tq.z) - qz;
  if (rx * rx + ry * ry + rz * rz > max_dist_sq_d) return false;  // DistanceRejector on the FP64 residual (rejector.hpp:24)
  // weight and residual in the SOURCE frame (D = R^T M R, rs = R^T r): see gicp_precision_source
  if (FACTOR == 0) {
    D = Sym3{1.0, 0.0, 0.0, 1.0, 0.0, 1.0};
  } else if (FACTOR == 1) {
    const float4 nrm = *t1;
    D = plane_weight_source(R, nrm.x, nrm.y, nrm.z);
  } else {
    D = gicp_precision_source(R, *sA, *sB, *t1, *t2);
  }
  rs[0] = R[0] * rx + R[3] * ry + R[6] * rz;
  rs[1] = R[1] * rx + R[4] * ry + R[7] * rz;
  rs[2] = R[2] * rx + R[5] * ry + R[8] * rz;
  p[0] = csx + sx;
  p[1] = csy + sy;
  p[2] = csz + sz;
  return true;
}

/// One accepted-or-rejected correspondence of `linearize`, evaluated exactly as factor_reduce_kernel does it:
///   sp        source point, FP32, relative to the source centre (csx, csy, csz)
///   tq        matched target point, FP32, relative to the target centre
///   (tpx, tpy, tpz) = R c_s + t - c_t : the translation with both centres folded in (FP64)
///   sA, sB    source covariance (GICP);  t1, t2 = target normal, - (point-to-plane) or target covariance (GICP): pointers,
///             read only by the factor that needs them and only for accepted points (unused ones may be null)
/// Transform and residual in FP64, DistanceRejector on the FP64 residual (rejector.hpp:24: d2 > max rejects), weight and
/// residual carried to the SOURCE frame, sums into acc[0..27], inlier count into acc[28].  Returns false if rejected.
template <int FACTOR, int ROBUST>
SGB_HD bool point_linearize_source(const double* R, double tpx, double tpy, double tpz, double csx, double csy, double csz, double max_dist_sq_d,
                                   double robust_c, const float4& sp, const float4* sA, const float4* sB, const float4& tq, const float4* t1,
                                   const float4* t2, double* acc) {
  Sym3 D;
  double rs[3], p[3];
  if (!point_weight_source<FACTOR>(R, tpx, tpy, tpz, csx, csy, csz, max_dist_sq_d, sp, sA, sB, tq, t1, t2, D, rs, p)) return false;
  accumulate_factor_source<ROBUST>(D, rs[0], rs[1], rs[2], p[0], p[1], p[2], robust_c, acc);
  acc[kAcc] += 1.0;
  return true;
}

/// One cached correspondence of `error` (reduction.hpp:55-62): residual at the trial pose R | t', GICP precision matrix
/// re-derived from the rotation of the LAST LINEARIZE (gicp_factor.hpp:81-89 keeps the cached mahalanobis), robust weight.
template <int FACTOR, int ROBUST>
SGB_HD double point_error(const double* R, double tpx, double tpy, double tpz, const double* Rlin, double robust_c, const float4& sp, const float4& sA,
                          const float4& sB, const float4& tq, const float4& t1, const float4& t2) {
  const double sx = sp.x, sy = sp.y, sz = sp.z;
  const double qx = R[0] * sx + R[1] * sy + R[2] * sz + tpx;
  const double qy = R[3] * sx + R[4] * sy + R[5] * sz + tpy;
  const double qz = R[6] * sx + R[7] * sy + R[8] * sz + tpz;
  const double rx = static_cast<double>(tq.x) - qx, ry = static_cast<double>(tq.y) - qy, rz = static_cast<double>(tq.z) - qz;
  double e;
  if (FACTOR == 0) {
    e = 0.5 * (rx * rx + ry * ry + rz * rz);
  } else if (FACTOR == 1) {
    const double ex = static_cast<double>(t1.x) * rx, ey = static_cast<double>(t1.y) * ry, ez = static_cast<double>(t1.z) * rz;
    e = 0.5 * (ex * ex + ey * ey + ez * ez);
  } else {
    const Sym3 M = gicp_precision(Rlin, sA, sB, t1, t2);
    const double mrx = M.xx * rx + M.xy * ry + M.xz * rz;
    const double mry = M.xy * rx + M.yy * ry + M.yz * rz;
    const double mrz = M.xz * rx + M.yz * ry + M.zz * rz;
    e = 0.5 * (rx * mrx + ry * mry + rz * mrz);
  }
  if (ROBUST == 1) {
    const double x = sqrt(e);
    e *= (x < robust_c ? 1.0 : robust_c / x);
  } else if (ROBUST == 2) {
    const double x = sqrt(e);
    e *= robust_c / (robust_c + x * x);
  }
  return e;
}

/// Unit vector spanning the kernel of the symmetric 3x3 t (row-major, rank 2 up to rounding): the longer of the cross products of
/// the column with the largest diagonal entry and the two other columns (extract_kernel of Eigen's computeDirect).
SGB_HD void sym3_kernel_vector(const double t[9], double v[3]) {
  int i0 = 0;
  if (fabs(t[4]) > fabs(t[0])) i0 = 1;
  if (fabs(t[8]) > fabs(t[i0 * 4])) i0 = 2;
  const int i1 = (i0 + 1) % 3, i2 = (i0 + 2) % 3;
  const double r[3] = {t[i0], t[3 + i0], t[6 + i0]}, a[3] = {t[i1], t[3 + i1], t[6 + i1]}, b[3] = {t[i2], t[3 + i2], t[6 + i2]};
  const double c0[3] = {r[1] * a[2] - r[2] * a[1], r[2] * a[0] - r[0] * a[2], r[0] * a[1] - r[1] * a[0]};
  const double c1[3] = {r[1] * b[2] - r[2] * b[1], r[2] * b[0] - r[0] * b[2], r[0] * b[1] - r[1] * b[0]};
  const double n0 = c0[0] * c0[0] + c0[1] * c0[1] + c0[2] * c0[2], n1 = c1[0] * c1[0] + c1[1] * c1[1] + c1[2] * c1[2];
  const double* c = n0 > n1 ? c0 : c1;
  const double inv = 1.0 / sqrt(n0 > n1 ? n0 : n1);
  v[0] = c[0] * inv;
  v[1] = c[1] * inv;
  v[2] = c[2] * inv;
}

/// Unit eigenvector of the smallest eigenvalue of a symmetric 3x3 (the only part of the decomposition the regularised covariance
/// and the normal need, normal_estimation.hpp:17-24,40-45).  Eigenvalues in closed form as Eigen's computeDirect computes them
/// (shift by the mean diagonal, scale by the largest entry, trigonometric roots).  Where a root is double, those formulas lose half
/// the digits of that root, so the eigenvector is taken from the MOST DISTINCT eigenvalue first, as computeDirect does:
///   * lambda_0 most distinct (planes): v = kernel of A - lambda_0 I, a rank-2 matrix;
///   * lambda_2 most distinct (lines, lambda_0 ~ lambda_1): u = kernel of A - lambda_2 I, then v = the smaller eigenvector of A
///     restricted to the plane orthogonal to u (a 2x2 problem solved by one rotation, atan2), so v is orthogonal to u by
///     construction.  When lambda_0 == lambda_1 that rotation is 0 and v is w = u x p of the plane's fixed basis (p, w).
/// Taking the kernel of A - lambda_min I directly instead fails on collinear neighbourhoods: that matrix has rank 1, lambda_min
/// is off by ~1e-8 lambda_2, and the cross products of its rows are rounding noise with components along the line.
/// Isotropic (all eigenvalues equal) or zero matrix: v = (1, 0, 0).
SGB_HD void smallest_eigenvector(double a00, double a01, double a02, double a11, double a12, double a22, double v[3]) {
  const double eps = 2.220446049250313e-16;
  const double shift = (a00 + a11 + a22) / 3.0;
  double m[9] = {a00 - shift, a01, a02, a01, a11 - shift, a12, a02, a12, a22 - shift};
  const double scale = fmax(fmax(fmax(fabs(m[0]), fabs(m[4])), fmax(fabs(m[8]), fabs(m[1]))), fmax(fabs(m[2]), fabs(m[5])));
  v[0] = 1.0;
  v[1] = 0.0;
  v[2] = 0.0;
  if (!(scale > 0.0)) return;
  for (int i = 0; i < 9; i++) m[i] /= scale;
  // computeRoots: ascending e0 <= e1 <= e2 of the shifted, scaled matrix
  const double c0 = m[0] * m[4] * m[8] + 2.0 * m[1] * m[2] * m[5] - m[0] * m[5] * m[5] - m[4] * m[2] * m[2] - m[8] * m[1] * m[1];
  const double c1 = m[0] * m[4] - m[1] * m[1] + m[0] * m[8] - m[2] * m[2] + m[4] * m[8] - m[5] * m[5];
  const double c2_over_3 = (m[0] + m[4] + m[8]) * (1.0 / 3.0);
  const double a_over_3 = fmax((c2_over_3 * c2_over_3 * 3.0 - c1) * (1.0 / 3.0), 0.0);
  const double half_b = 0.5 * (c0 + c2_over_3 * (2.0 * c2_over_3 * c2_over_3 - c1));
  const double q = fmax(a_over_3 * a_over_3 * a_over_3 - half_b * half_b, 0.0);
  const double rho = sqrt(a_over_3);
  const double theta = atan2(sqrt(q), half_b) * (1.0 / 3.0);
  const double cos_t = cos(theta), sin_t = sin(theta), sqrt3 = 1.7320508075688772;
  const double e0 = c2_over_3 - rho * (cos_t + sqrt3 * sin_t);
  const double e1 = c2_over_3 - rho * (cos_t - sqrt3 * sin_t);
  const double e2 = c2_over_3 + 2.0 * rho * cos_t;
  if (!(e2 - e0 > eps)) return;  // (numerically) isotropic: any direction is an eigenvector
  double t[9];
  if (e1 - e0 >= e2 - e1) {  // lambda_0 is the most distinct
    for (int i = 0; i < 9; i++) t[i] = m[i];
    t[0] -= e0;
    t[4] -= e0;
    t[8] -= e0;
    sym3_kernel_vector(t, v);
    return;
  }
  double u[3];
  for (int i = 0; i < 9; i++) t[i] = m[i];
  t[0] -= e2;
  t[4] -= e2;
  t[8] -= e2;
  sym3_kernel_vector(t, u);
  // orthonormal basis (p, w) of the plane orthogonal to u: p = u x (the axis u is least aligned with), w = u x p
  const double ax = fabs(u[0]), ay = fabs(u[1]), az = fabs(u[2]);
  double p[3];
  if (ax <= ay && ax <= az) {
    p[0] = 0.0; p[1] = u[2]; p[2] = -u[1];  // u x e_x
  } else if (ay <= az) {
    p[0] = -u[2]; p[1] = 0.0; p[2] = u[0];  // u x e_y
  } else {
    p[0] = u[1]; p[1] = -u[0]; p[2] = 0.0;  // u x e_z
  }
  const double ip = 1.0 / sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
  p[0] *= ip; p[1] *= ip; p[2] *= ip;
  const double w[3] = {u[1] * p[2] - u[2] * p[1], u[2] * p[0] - u[0] * p[2], u[0] * p[1] - u[1] * p[0]};
  // 2x2 restriction [[s_pp, s_pw], [s_pw, s_ww]]; its larger eigenvector is at angle phi = atan2(2 s_pw, s_pp - s_ww) / 2
  const double mp[3] = {m[0] * p[0] + m[1] * p[1] + m[2] * p[2], m[3] * p[0] + m[4] * p[1] + m[5] * p[2], m[6] * p[0] + m[7] * p[1] + m[8] * p[2]};
  const double mw[3] = {m[0] * w[0] + m[1] * w[1] + m[2] * w[2], m[3] * w[0] + m[4] * w[1] + m[5] * w[2], m[6] * w[0] + m[7] * w[1] + m[8] * w[2]};
  const double s_pp = p[0] * mp[0] + p[1] * mp[1] + p[2] * mp[2], s_ww = w[0] * mw[0] + w[1] * mw[1] + w[2] * mw[2];
  const double s_pw = 0.5 * ((w[0] * mp[0] + w[1] * mp[1] + w[2] * mp[2]) + (p[0] * mw[0] + p[1] * mw[1] + p[2] * mw[2]));
  const double phi = 0.5 * atan2(2.0 * s_pw, s_pp - s_ww);
  const double cp = cos(phi), sp = sin(phi);
  // the smaller eigenvector is the larger one turned by 90 degrees: -sin(phi) p + cos(phi) w
  for (int i = 0; i < 3; i++) v[i] = cp * w[i] - sp * p[i];
}

/// Where compact sum k (0..27, 28 = inlier count) goes in the expanded output  H (6x6 row-major) | b (6) | e | inliers:
/// p0 always, p1 too when the function returns 2 (the mirrored entry of the symmetric H).
SGB_HD int expand_positions(int k, int& p0, int& p1) {
  p1 = -1;
  if (k < 6) {  // H_rr upper triangle: (0,0)(0,1)(0,2)(1,1)(1,2)(2,2)
    const int r = k < 3 ? 0 : (k < 5 ? 1 : 2);
    const int c = k < 3 ? k : (k < 5 ? k - 2 : 2);
    p0 = r * 6 + c;
    p1 = c * 6 + r;
    return 2;
  }
  if (k < 15) {  // H_rt 3x3 row-major -> rows 0..2, cols 3..5 (+ transpose)
    const int r = (k - 6) / 3, c = (k - 6) % 3;
    p0 = r * 6 + 3 + c;
    p1 = (3 + c) * 6 + r;
    return 2;
  }
  if (k < 21) {  // H_tt upper triangle
    const int kk = k - 15;
    const int r = kk < 3 ? 0 : (kk < 5 ? 1 : 2);
    const int c = kk < 3 ? kk : (kk < 5 ? kk - 2 : 2);
    p0 = (3 + r) * 6 + 3 + c;
    p1 = (3 + c) * 6 + 3 + r;
    return 2;
  }
  if (k < 27) {
    p0 = 36 + (k - 21);  // b
    return 1;
  }
  p0 = k == 27 ? 42 : 43;  // e, inlier count
  return 1;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// The optimiser of batched align() (batch_step_kernel, sgb_batch.cu): GaussNewtonOptimizer / LevenbergMarquardtOptimizer of
// small_gicp_b200/host/include/small_gicp_b200/registration.hpp as a per-member state machine, one call per round.  The solve, the
// exponential and the pose product are written operation for operation like solve_ldlt / so3_exp / se3_exp / Isometry3d::operator* of
// core.hpp: compiled for the host without FMA contraction (tests/host_step) they give the same bits.  The installed host mirror must not
// depend on csrc/, so core.hpp keeps its own definitions; a change to either copy must be made to both.
// Matrices are column-major like core.hpp's Mat: A(r, c) = A[c * rows + r].  Poses are 4x4 (Isometry3d::data()).
// ---------------------------------------------------------------------------------------------------------------------------------

/// x = A^-1 rhs for a symmetric 6x6 A (destroyed) by LDL^T with diagonal pivoting; zero pivots give zero components (core.hpp solve_ldlt).
SGB_HD void solve_ldlt6(double* A, const double* rhs, double* x) {
  constexpr int n = 6;
  int perm[n];
  for (int i = 0; i < n; i++) perm[i] = i;
  for (int k = 0; k < n; k++) {
    int piv = k;
    for (int i = k + 1; i < n; i++)
      if (fabs(A[i * n + i]) > fabs(A[piv * n + piv])) piv = i;
    if (piv != k) {
      for (int j = 0; j < n; j++) {
        const double t = A[j * n + k];
        A[j * n + k] = A[j * n + piv];
        A[j * n + piv] = t;
      }
      for (int i = 0; i < n; i++) {
        const double t = A[k * n + i];
        A[k * n + i] = A[piv * n + i];
        A[piv * n + i] = t;
      }
      const int t = perm[k];
      perm[k] = perm[piv];
      perm[piv] = t;
    }
    for (int j = 0; j < k; j++) A[k * n + k] -= A[j * n + k] * A[j * n + k] * A[j * n + j];
    for (int i = k + 1; i < n; i++) {
      double s = A[k * n + i];
      for (int j = 0; j < k; j++) s -= A[j * n + i] * A[j * n + k] * A[j * n + j];
      A[k * n + i] = A[k * n + k] != 0.0 ? s / A[k * n + k] : 0.0;
    }
  }
  double y[n];
  for (int i = 0; i < n; i++) y[i] = rhs[perm[i]];
  for (int i = 0; i < n; i++)
    for (int j = 0; j < i; j++) y[i] -= A[j * n + i] * y[j];
  for (int i = 0; i < n; i++) y[i] = fabs(A[i * n + i]) > 0.0 ? y[i] / A[i * n + i] : 0.0;
  for (int i = n - 1; i >= 0; i--)
    for (int j = i + 1; j < n; j++) y[i] -= A[i * n + j] * y[j];
  for (int i = 0; i < n; i++) x[perm[i]] = y[i];
}

/// (H + lambda I) delta = -b  (detail::damped_step of registration.hpp)
SGB_HD void damped_step6(const double* H, const double* b, double lambda, double* delta) {
  double A[36], rhs[6];
  for (int i = 0; i < 36; i++) A[i] = H[i];
  for (int i = 0; i < 6; i++) A[i * 6 + i] += lambda;
  for (int i = 0; i < 6; i++) rhs[i] = -b[i];
  solve_ldlt6(A, rhs, delta);
}

/// out = A v for a 3x3 A (Mat's product: each entry summed from 0 in k order)
SGB_HD void mat3_vec(const double* A, const double* v, double* out) {
  for (int r = 0; r < 3; r++) out[r] = 0.0;
  for (int k = 0; k < 3; k++)
    for (int r = 0; r < 3; r++) out[r] += A[k * 3 + r] * v[k];
}

/// rotation matrix of a rotation vector through the unit quaternion (core.hpp so3_exp)
SGB_HD void so3_exp3(const double* omega, double* R) {
  double th2 = 0.0;
  for (int i = 0; i < 3; i++) th2 += omega[i] * omega[i];
  double im, re;
  if (th2 < 1e-10) {
    const double th4 = th2 * th2;
    im = 0.5 - th2 / 48.0 + th4 / 3840.0;
    re = 1.0 - th2 / 8.0 + th4 / 384.0;
  } else {
    const double th = sqrt(th2);
    im = sin(0.5 * th) / th;
    re = cos(0.5 * th);
  }
  const double w = re, x = im * omega[0], y = im * omega[1], z = im * omega[2];
  R[0] = 1.0 - 2.0 * (y * y + z * z);
  R[3] = 2.0 * (x * y - z * w);
  R[6] = 2.0 * (x * z + y * w);
  R[1] = 2.0 * (x * y + z * w);
  R[4] = 1.0 - 2.0 * (x * x + z * z);
  R[7] = 2.0 * (y * z - x * w);
  R[2] = 2.0 * (x * z - y * w);
  R[5] = 2.0 * (y * z + x * w);
  R[8] = 1.0 - 2.0 * (x * x + y * y);
}

/// 4x4 pose of a twist [rx ry rz tx ty tz] (core.hpp se3_exp)
SGB_HD void se3_exp6(const double* a, double* T) {
  const double* omega = a;
  const double* v = a + 3;
  double th2 = 0.0;
  for (int i = 0; i < 3; i++) th2 += omega[i] * omega[i];
  const double th = sqrt(th2);
  double R[9], t[3];
  so3_exp3(omega, R);
  if (th < 1e-10) {
    mat3_vec(R, v, t);
  } else {
    double W[9] = {0.0, omega[2], -omega[1], -omega[2], 0.0, omega[0], omega[1], -omega[0], 0.0};  // skew(omega)
    double WW[9];
    for (int i = 0; i < 9; i++) WW[i] = 0.0;
    for (int c = 0; c < 3; c++)
      for (int k = 0; k < 3; k++)
        for (int r = 0; r < 3; r++) WW[c * 3 + r] += W[k * 3 + r] * W[c * 3 + k];
    const double s1 = (1.0 - cos(th)) / th2, s2 = (th - sin(th)) / (th2 * th);
    double V[9];
    for (int i = 0; i < 9; i++) V[i] = ((i % 4 == 0) ? 1.0 : 0.0) + W[i] * s1;  // Identity() + W * s1
    for (int i = 0; i < 9; i++) V[i] = V[i] + WW[i] * s2;
    mat3_vec(V, v, t);
  }
  for (int c = 0; c < 3; c++) {
    for (int r = 0; r < 3; r++) T[c * 4 + r] = R[c * 3 + r];
    T[c * 4 + 3] = 0.0;
  }
  for (int r = 0; r < 3; r++) T[12 + r] = t[r];
  T[15] = 1.0;
}

/// out = A B for 4x4 poses (core.hpp Isometry3d::operator*: the full product, then the last row reset)
SGB_HD void pose_mul(const double* A, const double* B, double* out) {
  for (int i = 0; i < 16; i++) out[i] = 0.0;
  for (int c = 0; c < 4; c++)
    for (int k = 0; k < 4; k++) {
      const double b = B[c * 4 + k];
      for (int r = 0; r < 4; r++) out[c * 4 + r] += A[k * 4 + r] * b;
    }
  out[3] = out[7] = out[11] = 0.0;
  out[15] = 1.0;
}

/// TerminationCriteria::converged: |delta_rot| <= rotation_eps && |delta_trans| <= translation_eps
SGB_HD bool step_converged(const double* d, double rotation_eps, double translation_eps) {
  double r = 0.0, t = 0.0;
  for (int i = 0; i < 3; i++) r += d[i] * d[i];
  for (int i = 3; i < 6; i++) t += d[i] * d[i];
  return sqrt(r) <= rotation_eps && sqrt(t) <= translation_eps;
}

/// What the optimiser of one batched align() needs besides the reduction (sgb_align_options of include/sgicp_b200.h).
struct AlignOptions {
  int lm;  // 0: Gauss-Newton, 1: Levenberg-Marquardt
  int max_iterations, max_inner_iterations;
  double gn_lambda, init_lambda, lambda_factor;
  double rotation_eps, translation_eps;
  double dof_mask[6];  // RestrictDoFFactor: H(i,i) += 1e9 |mask_i - 1| (all ones: + 0, i.e. NullFactor)
};

/// next round of a member: linearize at T, error() at the candidate (LM), or nothing
enum : int { kPhaseLinearize = 0, kPhaseTrial = 1, kPhaseDone = 2 };

/// One member's optimiser between rounds.  T, converged, iterations, H, b, e and inliers are its RegistrationResult so far.
struct MemberState {
  double T[16];     // current pose
  double cand[16];  // LM: candidate pose of the pending trial
  double delta[6];  // LM: increment of the pending trial
  double H[36], b[6], e, inliers;  // last linearize (H with the RestrictDoFFactor term); e = LM's e / the result's error
  double lambda;
  int phase, it, trial, converged, iterations;
};

SGB_HHD void align_init(const AlignOptions& o, const double* T0, MemberState& s) {
  for (int i = 0; i < 16; i++) s.T[i] = s.cand[i] = T0[i];
  for (int i = 0; i < 6; i++) s.delta[i] = s.b[i] = 0.0;
  for (int i = 0; i < 36; i++) s.H[i] = 0.0;
  s.e = s.inliers = 0.0;
  s.lambda = o.init_lambda;
  s.phase = o.max_iterations > 0 ? kPhaseLinearize : kPhaseDone;
  s.it = s.trial = s.converged = s.iterations = 0;
}

SGB_HD void lm_propose(MemberState& s) {
  damped_step6(s.H, s.b, s.lambda, s.delta);
  double E[16];
  se3_exp6(s.delta, E);
  pose_mul(s.T, E, s.cand);
}

/// the outer iteration s.it is over: the next one, unless converged or out of iterations
SGB_HD void end_iteration(const AlignOptions& o, MemberState& s) {
  s.iterations = s.it;
  s.it++;
  s.phase = (s.it < o.max_iterations && !s.converged) ? kPhaseLinearize : kPhaseDone;
}

/// out44 = H | b | e | inliers of the linearize at s.T
SGB_HD void align_after_linearize(const AlignOptions& o, MemberState& s, const double* out44) {
  for (int i = 0; i < 36; i++) s.H[i] = out44[i];  // symmetric: row- and column-major agree
  for (int i = 0; i < 6; i++) s.H[i * 6 + i] += 1e9 * fabs(o.dof_mask[i] - 1.0);
  for (int i = 0; i < 6; i++) s.b[i] = out44[36 + i];
  s.e = out44[42];
  s.inliers = out44[43];
  if (!o.lm) {
    double d[6], E[16], T[16];
    damped_step6(s.H, s.b, o.gn_lambda, d);
    s.converged = step_converged(d, o.rotation_eps, o.translation_eps);
    se3_exp6(d, E);
    pose_mul(s.T, E, T);
    for (int i = 0; i < 16; i++) s.T[i] = T[i];
    end_iteration(o, s);
    return;
  }
  s.trial = 0;
  if (o.max_inner_iterations <= 0) {  // no trial: nothing accepted
    s.iterations = s.it;
    s.phase = kPhaseDone;
    return;
  }
  lm_propose(s);
  s.phase = kPhaseTrial;
}

/// candidate_e = error() at s.cand with the correspondences of the last linearize (LM)
SGB_HD void align_after_error(const AlignOptions& o, MemberState& s, double candidate_e) {
  if (candidate_e <= s.e) {
    s.converged = step_converged(s.delta, o.rotation_eps, o.translation_eps);
    for (int i = 0; i < 16; i++) s.T[i] = s.cand[i];
    s.lambda /= o.lambda_factor;
    s.e = candidate_e;
    end_iteration(o, s);
    return;
  }
  s.lambda *= o.lambda_factor;
  if (++s.trial < o.max_inner_iterations) {
    lm_propose(s);
    return;
  }
  s.iterations = s.it;  // every trial rejected: the reference breaks out of the outer loop
  s.phase = kPhaseDone;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Graduated non-convexity (sgb_align_batch_gnc, the gnc_* kernels in sgb_batch.cu; DESIGN.md §11 "Graduated non-convexity"): the
// closed-form weight of a point of squared residual r2 under the surrogate of shape mu, and the mu schedule.  Every operation is an
// explicitly rounded FP64 one in a fixed order, so nothing is contracted into an FMA and numpy reproduces every bit (tests/np_gnc.py;
// compiled for the host in tests/host_gnc, where the plain operators are built without contraction).
// ---------------------------------------------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
SGB_HD double rn_add(double a, double b) { return __dadd_rn(a, b); }
SGB_HD double rn_sub(double a, double b) { return __dsub_rn(a, b); }
SGB_HD double rn_mul(double a, double b) { return __dmul_rn(a, b); }
SGB_HD double rn_div(double a, double b) { return __ddiv_rn(a, b); }
SGB_HD double rn_sqrt(double a) { return __dsqrt_rn(a); }
#else
SGB_HD double rn_add(double a, double b) { return a + b; }
SGB_HD double rn_sub(double a, double b) { return a - b; }
SGB_HD double rn_mul(double a, double b) { return a * b; }
SGB_HD double rn_div(double a, double b) { return a / b; }
SGB_HD double rn_sqrt(double a) { return std::sqrt(a); }
#endif

enum : int { kGncGemanMcClure = 0, kGncTls = 1 };  // sgb_gnc_kind
constexpr double kGncFactor = 1.4;                  // the annealing factor of Yang et al. (RA-L 2020)

/// The weight of a point with squared residual r2 (>= 0 up to rounding) under the surrogate of shape mu, noise bound c2:
///   Geman-McClure  (mu c2 / (r2 + mu c2))^2
///   TLS            1 if r2 <= mu / (mu + 1) c2, 0 if r2 >= (mu + 1) / mu c2, else min(max(sqrt(c2) / sqrt(r2) sqrt(mu (mu + 1)) - mu, 0), 1)
/// (the clamp only catches the rounding of the middle branch at its two edges, where it is 1 and 0).
template <int KIND>
SGB_HD double gnc_weight(double r2, double mu, double c2) {
  if constexpr (KIND == kGncGemanMcClure) {
    const double a = rn_mul(mu, c2);
    const double q = rn_div(a, rn_add(r2, a));
    return rn_mul(q, q);
  } else {
    const double mu1 = rn_add(mu, 1.0);
    if (r2 <= rn_mul(rn_div(mu, mu1), c2)) return 1.0;
    if (r2 >= rn_mul(rn_div(mu1, mu), c2)) return 0.0;
    const double g = rn_sub(rn_mul(rn_div(rn_sqrt(c2), rn_sqrt(r2)), rn_sqrt(rn_mul(mu, mu1))), mu);
    return g < 0.0 ? 0.0 : (g > 1.0 ? 1.0 : g);
  }
}

/// One member's GNC between stages.  r2max: the largest r^2 > 0 of stage 0's reweighting linearize (0: none), kept as the bits of a
/// non-negative double so that atomicMax on them is an exact, order-free maximum.
struct GncState {
  double mu;          // the surrogate's shape of the current (after the loop: the last) stage
  double r2max;
  int stages;         // stages begun
  int last;           // the current stage is the member's last
  int ones;           // TLS without outliers (2 r2max <= c2): every weight of its only stage is 1
  unsigned not_binary;  // TLS: a weight of the current stage lies strictly between 0 and 1
  int iterations;     // the iterations of the member's finished stages
};

/// The start of a member's next stage: mu_0 from r2max at stage 0 (GM: 2 r2max / c2, at least 1; TLS: c2 / (2 r2max - c2), or none
/// without outliers), else the schedule's next mu (GM: max(mu / 1.4, 1); TLS: 1.4 mu).  The stage is the last when GM reaches mu = 1,
/// TLS has no outliers, or it is stage max_stages - 1; TLS also ends at a stage whose weights are all binary (decided after them).
SGB_HD void gnc_stage_begin(int kind, double c2, int max_stages, GncState& g) {
  if (g.stages == 0) {
    const double t = rn_mul(2.0, g.r2max);
    if (kind == kGncGemanMcClure) {
      g.mu = rn_div(t, c2);
      if (g.mu <= 1.0) g.mu = 1.0;
    } else if (t <= c2) {
      g.mu = 0.0;
      g.ones = 1;
    } else {
      g.mu = rn_div(c2, rn_sub(t, c2));
    }
  } else if (kind == kGncGemanMcClure) {
    const double m = rn_div(g.mu, kGncFactor);
    g.mu = m > 1.0 ? m : 1.0;
  } else {
    g.mu = rn_mul(kGncFactor, g.mu);
  }
  g.last = g.ones || (kind == kGncGemanMcClure && g.mu == 1.0) || g.stages == max_stages - 1;
  g.stages++;
  g.not_binary = 0u;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Joint window registration (sgb_align_joint, joint_step_kernel in sgb_batch.cu; DESIGN.md §11 "Joint windows").  The frames X_k of a
// window are solved together against every edge (i, j) of the window, each edge a pair member at T_e = X_j^-1 X_i.  The functions below
// are run by every thread of one CTA (tid of nt threads, CTA barriers between phases); compiled for the host (tests/host_joint) they run
// with tid = 0, nt = 1 and no barrier.
// ---------------------------------------------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
#define SGB_CTA_SYNC() __syncthreads()
#else
#define SGB_CTA_SYNC() ((void)0)
#endif

constexpr int kJointMaxFrames = 32;
constexpr int kJointMaxN = 6 * kJointMaxFrames;

/// position of entry (r, c) of a symmetric n x n matrix stored as its packed lower triangle, row after row
SGB_HD int packed_index(int r, int c) { return r >= c ? r * (r + 1) / 2 + c : c * (c + 1) / 2 + r; }

/// solve_ldlt6 for a symmetric n x n A given as its packed lower triangle L (destroyed), n <= kJointMaxN: the same diagonal pivoting and
/// the same operations in the same order for every entry (each entry's j-sum sequential), so n = 6 gives solve_ldlt6's bits.  The rows of
/// each column are spread over the threads; the back substitution, whose order chains every entry, is thread 0's.  perm [n] and y [n] are
/// scratch of the CTA (shared memory on the device).  solve_ldlt6 swaps whole rows and columns; only the lower triangle is ever read, and
/// the symmetric swap below moves its entries exactly as the full swap does (the trailing block is still symmetric when it is swapped).
SGB_HD void solve_ldlt_n(int n, double* L, const double* rhs, double* x, int* perm, double* y, int tid, int nt) {
  for (int i = tid; i < n; i += nt) perm[i] = i;
  SGB_CTA_SYNC();
  for (int k = 0; k < n; k++) {
    int piv = k;
    for (int i = k + 1; i < n; i++)
      if (fabs(L[packed_index(i, i)]) > fabs(L[packed_index(piv, piv)])) piv = i;
    SGB_CTA_SYNC();  // every thread has read the diagonal before it is swapped
    if (piv != k) {
      for (int m = tid; m < n; m += nt) {
        int a, b;
        if (m < k) {
          a = packed_index(k, m), b = packed_index(piv, m);
        } else if (m == k) {
          a = packed_index(k, k), b = packed_index(piv, piv);
        } else if (m < piv) {
          a = packed_index(m, k), b = packed_index(piv, m);
        } else if (m > piv) {
          a = packed_index(m, k), b = packed_index(m, piv);
        } else {
          continue;  // (piv, k) maps onto itself
        }
        const double t = L[a];
        L[a] = L[b];
        L[b] = t;
      }
      if (tid == 0) {
        const int t = perm[k];
        perm[k] = perm[piv];
        perm[piv] = t;
      }
      SGB_CTA_SYNC();
    }
    for (int i = k + tid; i < n; i += nt) {  // the sums of column k, each in place (the divisions wait for the new pivot)
      const int ik = packed_index(i, k);
      double s = L[ik];
      for (int j = 0; j < k; j++) s -= L[packed_index(i, j)] * L[packed_index(k, j)] * L[packed_index(j, j)];
      L[ik] = s;
    }
    SGB_CTA_SYNC();
    const double d = L[packed_index(k, k)];
    for (int i = k + 1 + tid; i < n; i += nt) {
      const int ik = packed_index(i, k);
      L[ik] = d != 0.0 ? L[ik] / d : 0.0;
    }
    SGB_CTA_SYNC();
  }
  for (int i = tid; i < n; i += nt) y[i] = rhs[perm[i]];
  SGB_CTA_SYNC();
  for (int j = 0; j < n; j++) {  // y[i] -= L(i, j) y[j] for j = 0 .. i - 1 in that order, column by column
    for (int i = j + 1 + tid; i < n; i += nt) y[i] -= L[packed_index(i, j)] * y[j];
    SGB_CTA_SYNC();
  }
  for (int i = tid; i < n; i += nt) {
    const double d = L[packed_index(i, i)];
    y[i] = fabs(d) > 0.0 ? y[i] / d : 0.0;
  }
  SGB_CTA_SYNC();
  if (tid == 0)
    for (int i = n - 1; i >= 0; i--)
      for (int j = i + 1; j < n; j++) y[i] -= L[packed_index(j, i)] * y[j];
  SGB_CTA_SYNC();
  for (int i = tid; i < n; i += nt) x[perm[i]] = y[i];
  SGB_CTA_SYNC();
}

/// inverse of a rigid 4x4 pose (column-major): R^T | -R^T t
SGB_HD void pose_inverse(const double* X, double* out) {
  for (int c = 0; c < 3; c++) {
    for (int r = 0; r < 3; r++) out[c * 4 + r] = X[r * 4 + c];
    out[c * 4 + 3] = 0.0;
  }
  for (int r = 0; r < 3; r++) out[12 + r] = -(X[r * 4 + 0] * X[12] + X[r * 4 + 1] * X[13] + X[r * 4 + 2] * X[14]);
  out[15] = 1.0;
}

/// the pose of edge (i, j): T_e = X_j^-1 X_i
SGB_HD void edge_pose(const double* Xi, const double* Xj, double* T) {
  double inv[16];
  pose_inverse(Xj, inv);
  pose_mul(inv, Xi, T);
}

/// A_e = -Ad(T_e^-1), 6x6 row-major, Ad(R, t) = [[R, 0], [[t]x R, R]] for twists [r; t]: the right perturbations of the frames move the
/// edge by delta_e = delta_i + A_e delta_j
SGB_HD void edge_adjoint(const double* T, double* A) {
  double inv[16];
  pose_inverse(T, inv);
  const double* t = inv + 12;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      const double R = inv[c * 4 + r];
      // ([t]x R)(r, c) = sum_k [t]x(r, k) R(k, c)
      const double tx = r == 0 ? t[1] * inv[c * 4 + 2] - t[2] * inv[c * 4 + 1]
                               : (r == 1 ? t[2] * inv[c * 4 + 0] - t[0] * inv[c * 4 + 2] : t[0] * inv[c * 4 + 1] - t[1] * inv[c * 4 + 0]);
      A[r * 6 + c] = -R;
      A[r * 6 + 3 + c] = 0.0;
      A[(3 + r) * 6 + c] = -tx;
      A[(3 + r) * 6 + 3 + c] = -R;
    }
}

/// One window's optimiser between rounds (beside MemberState: the scalars; the frames' poses, candidates and steps are arrays of the call).
struct WindowState {
  double e, inliers;  // summed over the window's edges at the last linearize (e: LM's e / the result's error)
  double lambda;
  int phase, it, trial, converged, iterations;
};

/// One window as the step sees it.  Frames 0 .. n_frames - 1 (local), free[k] = index of frame k among the free frames or -1 (fixed);
/// edges 0 .. n_edges - 1 in member order, edge q = cloud ei[q] against map ej[q] (local frames), sums [n_edges][44] = its H | b | e | inliers
/// of the last linearize.  X, cand: [n_frames][16]; delta: [6 n_free].  work: the CTA's scratch of joint_work_doubles(n_free) doubles.
struct JointWindow {
  int n_frames, n_free, n_edges;
  const int* free;
  const int *ei, *ej;
  const double* sums;
  double *X, *cand, *delta;
  WindowState* s;
  double* work;
};

SGB_HHD int joint_work_doubles(int n_free) {
  const int n = 6 * n_free;
  return n * (n + 1) / 2 + 3 * n + 36 * 3 + 6 + (n + 1) / 2 + 4;  // L | b | rhs | y | A, P, Q | c | perm (ints) | flags
}

SGB_HHD void joint_init(const AlignOptions& o, int n_free, int n_edges, WindowState& s) {
  s.e = s.inliers = 0.0;
  s.lambda = o.init_lambda;
  s.phase = o.max_iterations > 0 && n_free > 0 && n_edges > 0 ? kPhaseLinearize : kPhaseDone;
  s.it = s.trial = s.converged = s.iterations = 0;
}

/// L | b of the window from its edges' sums: H_ii += H_e, H_ij += H_e A_e, H_jj += A_e^T H_e A_e, b_i += b_e, b_j += A_e^T b_e for the free
/// frames among i, j, edge after edge in member order; then 1e9 |mask - 1| on every free frame's diagonal and lambda on every diagonal entry.
SGB_HD void joint_assemble(const AlignOptions& o, const JointWindow& w, double lambda, int tid, int nt) {
  const int n = 6 * w.n_free;
  double* L = w.work;
  double* b = L + n * (n + 1) / 2;
  double* A = b + 3 * n;
  double* P = A + 36;
  double* Q = P + 36;
  double* c = Q + 36;
  for (int k = tid; k < n * (n + 1) / 2 + n; k += nt) L[k] = 0.0;  // L and b are contiguous
  SGB_CTA_SYNC();
  for (int q = 0; q < w.n_edges; q++) {
    const int fi = w.free[w.ei[q]], fj = w.free[w.ej[q]];
    const double* H = w.sums + 44 * static_cast<size_t>(q);  // symmetric: row- and column-major agree
    if (fj >= 0) {
      if (tid == 0) {
        double T[16];
        edge_pose(w.X + 16 * w.ei[q], w.X + 16 * w.ej[q], T);
        edge_adjoint(T, A);
      }
      SGB_CTA_SYNC();
      for (int k = tid; k < 36; k += nt) {  // P = H A
        const int r = k / 6, cc = k % 6;
        double v = 0.0;
        for (int m = 0; m < 6; m++) v += H[r * 6 + m] * A[m * 6 + cc];
        P[k] = v;
      }
      SGB_CTA_SYNC();
      for (int k = tid; k < 42; k += nt) {  // Q = A^T P, c = A^T b
        if (k < 36) {
          const int r = k / 6, cc = k % 6;
          double v = 0.0;
          for (int m = 0; m < 6; m++) v += A[m * 6 + r] * P[m * 6 + cc];
          Q[k] = v;
        } else {
          const int r = k - 36;
          double v = 0.0;
          for (int m = 0; m < 6; m++) v += A[m * 6 + r] * H[36 + m];
          c[r] = v;
        }
      }
      SGB_CTA_SYNC();
    }
    for (int k = tid; k < 36 * 3 + 12; k += nt) {  // every target entry is one thread's
      if (k < 36) {
        const int r = k / 6, cc = k % 6;
        if (fi >= 0 && r >= cc) L[packed_index(6 * fi + r, 6 * fi + cc)] += H[r * 6 + cc];
      } else if (k < 72) {
        const int r = (k - 36) / 6, cc = (k - 36) % 6;
        if (fj >= 0 && r >= cc) L[packed_index(6 * fj + r, 6 * fj + cc)] += Q[r * 6 + cc];
      } else if (k < 108) {
        const int r = (k - 72) / 6, cc = (k - 72) % 6;
        if (fi >= 0 && fj >= 0) {
          if (fi > fj)
            L[packed_index(6 * fi + r, 6 * fj + cc)] += P[r * 6 + cc];  // H_ij = H_e A_e
          else
            L[packed_index(6 * fj + r, 6 * fi + cc)] += P[cc * 6 + r];  // H_ji = A_e^T H_e = P^T
        }
      } else if (k < 114) {
        if (fi >= 0) b[6 * fi + k - 108] += H[36 + k - 108];
      } else {
        if (fj >= 0) b[6 * fj + k - 114] += c[k - 114];
      }
    }
    SGB_CTA_SYNC();
  }
  for (int k = tid; k < n; k += nt) {
    const int d = packed_index(k, k);
    L[d] += 1e9 * fabs(o.dof_mask[k % 6] - 1.0);
  }
  SGB_CTA_SYNC();
  for (int k = tid; k < n; k += nt) L[packed_index(k, k)] += lambda;
  SGB_CTA_SYNC();
}

/// delta = (H + lambda I)^-1 (-b) over the window's free frames; returns whether every free frame's step meets the termination criteria
SGB_HD bool joint_solve(const AlignOptions& o, const JointWindow& w, double lambda, int tid, int nt) {
  const int n = 6 * w.n_free;
  joint_assemble(o, w, lambda, tid, nt);
  double* L = w.work;
  double* b = L + n * (n + 1) / 2;
  double* rhs = b + n;
  double* y = rhs + n;
  int* perm = reinterpret_cast<int*>(y + n + 36 * 3 + 6);
  int* flag = perm + n + (n & 1);
  for (int k = tid; k < n; k += nt) rhs[k] = -b[k];
  if (tid == 0) *flag = 1;
  SGB_CTA_SYNC();
  solve_ldlt_n(n, L, rhs, w.delta, perm, y, tid, nt);
  for (int f = tid; f < w.n_free; f += nt)
    if (!step_converged(w.delta + 6 * f, o.rotation_eps, o.translation_eps)) *flag = 0;
  SGB_CTA_SYNC();
  const bool conv = *flag != 0;
  SGB_CTA_SYNC();
  return conv;
}

/// out = X exp(delta_k) for the free frames, X for the fixed ones
SGB_HD void joint_update(const JointWindow& w, const double* X, double* out, int tid, int nt) {
  for (int k = tid; k < w.n_frames; k += nt) {
    const int f = w.free[k];
    if (f < 0) {
      for (int i = 0; i < 16; i++) out[16 * k + i] = X[16 * k + i];
      continue;
    }
    double E[16], T[16];
    se3_exp6(w.delta + 6 * f, E);
    pose_mul(X + 16 * k, E, T);
    for (int i = 0; i < 16; i++) out[16 * k + i] = T[i];
  }
  SGB_CTA_SYNC();
}

SGB_HD void joint_end_iteration(const AlignOptions& o, WindowState& s) {
  s.iterations = s.it;
  s.it++;
  s.phase = (s.it < o.max_iterations && !s.converged) ? kPhaseLinearize : kPhaseDone;
}

/// align_after_linearize for a window: the edges' sums of the linearize at X are in w.sums
SGB_HD void joint_after_linearize(const AlignOptions& o, JointWindow& w, int tid, int nt) {
  WindowState& s = *w.s;
  if (tid == 0) {
    double e = 0.0, inl = 0.0;
    for (int q = 0; q < w.n_edges; q++) {
      e += w.sums[44 * static_cast<size_t>(q) + 42];
      inl += w.sums[44 * static_cast<size_t>(q) + 43];
    }
    s.e = e;
    s.inliers = inl;
  }
  SGB_CTA_SYNC();
  if (!o.lm) {
    const bool conv = joint_solve(o, w, o.gn_lambda, tid, nt);
    joint_update(w, w.X, w.cand, tid, nt);
    for (int k = tid; k < 16 * w.n_frames; k += nt) w.X[k] = w.cand[k];
    if (tid == 0) {
      s.converged = conv;
      joint_end_iteration(o, s);
    }
    SGB_CTA_SYNC();
    return;
  }
  if (o.max_inner_iterations <= 0) {  // no trial: nothing accepted
    if (tid == 0) {
      s.trial = 0;
      s.iterations = s.it;
      s.phase = kPhaseDone;
    }
    SGB_CTA_SYNC();
    return;
  }
  const double lambda = s.lambda;
  joint_solve(o, w, lambda, tid, nt);
  joint_update(w, w.X, w.cand, tid, nt);
  if (tid == 0) {
    s.trial = 0;
    s.phase = kPhaseTrial;
  }
  SGB_CTA_SYNC();
}

/// align_after_error for a window: candidate_e = the window's error() at w.cand, summed over its edges in member order
SGB_HD void joint_after_error(const AlignOptions& o, JointWindow& w, double candidate_e, int tid, int nt) {
  WindowState& s = *w.s;
  const double e = s.e, lambda = s.lambda;
  const int trial = s.trial;
  SGB_CTA_SYNC();
  if (candidate_e <= e) {
    bool conv = true;
    for (int f = 0; f < w.n_free; f++) conv = conv && step_converged(w.delta + 6 * f, o.rotation_eps, o.translation_eps);
    for (int k = tid; k < 16 * w.n_frames; k += nt) w.X[k] = w.cand[k];
    if (tid == 0) {
      s.converged = conv;
      s.lambda = lambda / o.lambda_factor;
      s.e = candidate_e;
      joint_end_iteration(o, s);
    }
    SGB_CTA_SYNC();
    return;
  }
  const double next = lambda * o.lambda_factor;
  if (trial + 1 < o.max_inner_iterations) {
    joint_solve(o, w, next, tid, nt);
    joint_update(w, w.X, w.cand, tid, nt);
  }
  if (tid == 0) {
    s.lambda = next;
    s.trial = trial + 1;
    if (s.trial >= o.max_inner_iterations) {
      s.iterations = s.it;  // every trial rejected: the reference breaks out of the outer loop
      s.phase = kPhaseDone;
    }
  }
  SGB_CTA_SYNC();
}

}  // namespace sgb
