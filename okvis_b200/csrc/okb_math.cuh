// Per-thread math of the CUDA estimator path: kinematics, camera models, single-residual functors.
// Everything here is OKB_HD (host + device) so tests can also compile it for the host and compare it
// with the oracle without a GPU (tests/hostcheck); the product only ever calls it from kernels.
//
// The formulas follow the reference but are re-derived for the fused GPU pipeline (structure
// exploitation instead of generic matrix products):
//   reprojection: A = sqrtInfo * dproj/dp_C * C_CW (2x3);  J_lm = -A;  J_pose = A*[w I, -[p]x],
//     p = X_W - t_WS*w   (ReprojectionError.hpp(impl):87-242 multiplies the same factors as 4x4/4x6 matrices)
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/okvis_b200.h"

#if defined(__CUDACC__)
#define OKB_HD __host__ __device__ __forceinline__
#else
#define OKB_HD inline
#endif

namespace okb {

// ---------------------------------------------------------------- quaternions / rotations
// q = [x,y,z,w]; Hamilton product (Eigen convention used throughout OKVIS).
OKB_HD void qmul(const double* a, const double* b, double* o) {
  const double ax = a[0], ay = a[1], az = a[2], aw = a[3];
  const double bx = b[0], by = b[1], bz = b[2], bw = b[3];
  o[0] = aw * bx + ax * bw + ay * bz - az * by;
  o[1] = aw * by + ay * bw + az * bx - ax * bz;
  o[2] = aw * bz + az * bw + ax * by - ay * bx;
  o[3] = aw * bw - ax * bx - ay * by - az * bz;
}
OKB_HD void qinv(const double* q, double* o) {
  const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  const double i = 1.0 / n2;
  o[0] = -q[0] * i; o[1] = -q[1] * i; o[2] = -q[2] * i; o[3] = q[3] * i;
}
OKB_HD void qnormalize(double* q) {
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
// rotation matrix (row-major 3x3) of a quaternion, no normalisation (Eigen toRotationMatrix)
OKB_HD void q2R(const double* q, double* R) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w;
  const double txx = tx * x, txy = ty * x, txz = tz * x;
  const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
  R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}
OKB_HD double sinc(double x) {
  if (fabs(x) > 1e-6) return sin(x) / x;
  const double x2 = x * x, x4 = x2 * x2, x6 = x2 * x2 * x2;
  return 1.0 - x2 * (1.0 / 6.0) + x4 * (1.0 / 120.0) - x6 * (1.0 / 5040.0);
}
OKB_HD void deltaQ(const double* a, double* dq) {
  const double hn = 0.5 * sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
  const double s = sinc(hn) * 0.5;
  dq[0] = s * a[0]; dq[1] = s * a[1]; dq[2] = s * a[2]; dq[3] = cos(hn);
}
// 3x3 helpers, row-major
OKB_HD void mat3mul(const double* A, const double* B, double* C) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
}
OKB_HD void mat3Tmul(const double* A, const double* B, double* C) {  // A^T B
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[i * 3 + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
}
OKB_HD void mat3vec(const double* A, const double* v, double* o) {
#pragma unroll
  for (int i = 0; i < 3; ++i) o[i] = A[i * 3] * v[0] + A[i * 3 + 1] * v[1] + A[i * 3 + 2] * v[2];
}
OKB_HD void mat3Tvec(const double* A, const double* v, double* o) {
#pragma unroll
  for (int i = 0; i < 3; ++i) o[i] = A[i] * v[0] + A[3 + i] * v[1] + A[6 + i] * v[2];
}
OKB_HD void crossMx(const double* v, double* C) {
  C[0] = 0;     C[1] = -v[2]; C[2] = v[1];
  C[3] = v[2];  C[4] = 0;     C[5] = -v[0];
  C[6] = -v[1]; C[7] = v[0];  C[8] = 0;
}
OKB_HD void cross3(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
// rightJacobian (Forster et al.), series below 1e-4
OKB_HD void rightJacobian(const double* phi, double* R) {
  const double P = sqrt(phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2]);
  double X[9], X2[9];
  crossMx(phi, X);
  mat3mul(X, X, X2);
  double a, b;
  if (P < 1.0e-4) { a = -0.5; b = 1.0 / 6.0; }
  else { const double P2 = P * P; a = -(1.0 - cos(P)) / P2; b = (P - sin(P)) / (P2 * P); }
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = a * X[i] + b * X2[i];
  R[0] += 1.0; R[4] += 1.0; R[8] += 1.0;
}

// Pose = [t(3), q(4)].  plus: t += d[0:3]; q <- normalize(dq(d[3:6]) * q)
OKB_HD void pose_plus(const double* x, const double* d, double* o) {
  double q[4] = {x[3], x[4], x[5], x[6]};
  qnormalize(q);  // the reference builds a Transformation first, which normalises
  double dq[4], qn[4];
  deltaQ(d + 3, dq);
  qmul(dq, q, qn);
  qnormalize(qn);
  o[0] = x[0] + d[0]; o[1] = x[1] + d[1]; o[2] = x[2] + d[2];
  o[3] = qn[0]; o[4] = qn[1]; o[5] = qn[2]; o[6] = qn[3];
}
// minus(x, xpd): [t' - t; 2 vec(q' * q^-1)]
OKB_HD void pose_minus(const double* x, const double* xpd, double* d) {
  d[0] = xpd[0] - x[0]; d[1] = xpd[1] - x[1]; d[2] = xpd[2] - x[2];
  double qi[4], dq[4];
  qinv(x + 3, qi);
  qmul(xpd + 3, qi, dq);
  d[3] = 2 * dq[0]; d[4] = 2 * dq[1]; d[5] = 2 * dq[2];
}

// symmetric 3x3 stored as [xx, xy, xz, yy, yz, zz]
// Cholesky R = L L^T (L lower: l00,l10,l11,l20,l21,l22).  Returns false on a non-positive pivot.
OKB_HD bool chol3(const double* S, double* L) {
  double x = S[0];
  if (!(x > 0.0)) return false;
  L[0] = sqrt(x);
  L[1] = S[1] / L[0];
  L[3] = S[2] / L[0];
  x = S[3] - L[1] * L[1];
  if (!(x > 0.0)) return false;
  L[2] = sqrt(x);
  L[4] = (S[4] - L[3] * L[1]) / L[2];
  x = S[5] - L[3] * L[3] - L[4] * L[4];
  if (!(x > 0.0)) return false;
  L[5] = sqrt(x);
  return true;
}
// inverse of lower-triangular L (same packing)
OKB_HD void linv3(const double* L, double* Li) {
  Li[0] = 1.0 / L[0];
  Li[2] = 1.0 / L[2];
  Li[5] = 1.0 / L[5];
  Li[1] = -L[1] * Li[0] * Li[2];
  Li[4] = -L[4] * Li[2] * Li[5];
  Li[3] = -(L[3] * Li[0] + L[4] * Li[1]) * Li[5];
}
// symmetric 3x3 eigenvalues (ascending), closed form (trigonometric) with Jacobi polish for accuracy
OKB_HD void eig3sym(const double* S, double* ev) {
  double a[9] = {S[0], S[1], S[2], S[1], S[3], S[4], S[2], S[4], S[5]};
  for (int sweep = 0; sweep < 30; ++sweep) {
    const double off = a[1] * a[1] + a[2] * a[2] + a[5] * a[5];
    if (off < 1e-300) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        const double apq = a[p * 3 + q];
        if (fabs(apq) < 1e-300) continue;
        const double theta = (a[q * 3 + q] - a[p * 3 + p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) {
          const double akp = a[k * 3 + p], akq = a[k * 3 + q];
          a[k * 3 + p] = c * akp - s * akq; a[k * 3 + q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; ++k) {
          const double apk = a[p * 3 + k], aqk = a[q * 3 + k];
          a[p * 3 + k] = c * apk - s * aqk; a[q * 3 + k] = s * apk + c * aqk;
        }
      }
  }
  double e0 = a[0], e1 = a[4], e2 = a[8], t;
  if (e0 > e1) { t = e0; e0 = e1; e1 = t; }
  if (e1 > e2) { t = e1; e1 = e2; e2 = t; }
  if (e0 > e1) { t = e0; e0 = e1; e1 = t; }
  ev[0] = e0; ev[1] = e1; ev[2] = e2;
}

// closed-form (trigonometric) eigenvalues of a symmetric 3x3, ascending; branch-light for kernels
OKB_HD void eig3sym_closed(const double* S, double* ev) {
  const double a00 = S[0], a01 = S[1], a02 = S[2], a11 = S[3], a12 = S[4], a22 = S[5];
  const double p1 = a01 * a01 + a02 * a02 + a12 * a12;
  const double q = (a00 + a11 + a22) / 3.0;
  const double b00 = a00 - q, b11 = a11 - q, b22 = a22 - q;
  const double p2 = b00 * b00 + b11 * b11 + b22 * b22 + 2.0 * p1;
  if (!(p2 > 0.0)) { ev[0] = ev[1] = ev[2] = q; return; }
  const double p = sqrt(p2 / 6.0);
  const double ip = 1.0 / p;
  const double c00 = b00 * ip, c01 = a01 * ip, c02 = a02 * ip, c11 = b11 * ip, c12 = a12 * ip, c22 = b22 * ip;
  double r = 0.5 * (c00 * (c11 * c22 - c12 * c12) - c01 * (c01 * c22 - c12 * c02) + c02 * (c01 * c12 - c11 * c02));
  r = fmin(1.0, fmax(-1.0, r));
  const double phi = acos(r) / 3.0;
  const double e2 = q + 2.0 * p * cos(phi);
  const double e0 = q + 2.0 * p * cos(phi + 2.0943951023931953);
  ev[0] = e0; ev[2] = e2; ev[1] = 3.0 * q - e0 - e2;
}

// ---------------------------------------------------------------- camera models
struct CamIntr {  // compact per-slot copy of okb_camera
  double fu, fv, cu, cv;
  double k[8];
  int model;
};
OKB_HD void cam_load(const okb_camera& c, CamIntr& o) {
  o.fu = c.fu; o.fv = c.fv; o.cu = c.cu; o.cv = c.cv; o.model = c.model;
#pragma unroll
  for (int i = 0; i < 8; ++i) o.k[i] = c.dist[i];
}

// Distortion model of a projection: one of OKB_DIST_* fixes it at compile time, kDistAny switches on CamIntr::model
// at run time (unknown models project as OKB_DIST_NONE).  Kernels whose launch has one model across all cameras
// instantiate that model and carry no registers for the others.
constexpr int kDistAny = -1;

// distortion of the normalised point u -> d and (optionally) its 2x2 Jacobian Jd (row-major).
// Returns false where the reference's distort() fails (radtan8, rho > 9); outputs are then zero.
template <bool WANT_J, int MODEL = kDistAny>
OKB_HD bool distort(const CamIntr& c, double u0, double u1, double* d, double* Jd) {
  if constexpr (MODEL == kDistAny) {
    switch (c.model) {
      case OKB_DIST_RADTAN: return distort<WANT_J, OKB_DIST_RADTAN>(c, u0, u1, d, Jd);
      case OKB_DIST_EQUIDISTANT: return distort<WANT_J, OKB_DIST_EQUIDISTANT>(c, u0, u1, d, Jd);
      case OKB_DIST_RADTAN8: return distort<WANT_J, OKB_DIST_RADTAN8>(c, u0, u1, d, Jd);
      default: return distort<WANT_J, OKB_DIST_NONE>(c, u0, u1, d, Jd);
    }
  } else if constexpr (MODEL == OKB_DIST_RADTAN) {
    const double k1 = c.k[0], k2 = c.k[1], p1 = c.k[2], p2 = c.k[3];
    const double mx = u0 * u0, my = u1 * u1, mxy = u0 * u1, rho = mx + my;
    const double rad = k1 * rho + k2 * rho * rho;
    d[0] = u0 + u0 * rad + 2.0 * p1 * mxy + p2 * (rho + 2.0 * mx);
    d[1] = u1 + u1 * rad + 2.0 * p2 * mxy + p1 * (rho + 2.0 * my);
    if (WANT_J) {
      Jd[0] = 1 + rad + k1 * 2.0 * mx + k2 * rho * 4 * mx + 2.0 * p1 * u1 + 6 * p2 * u0;
      Jd[2] = k1 * 2.0 * u0 * u1 + k2 * 4 * rho * u0 * u1 + p1 * 2.0 * u0 + 2.0 * p2 * u1;
      Jd[1] = Jd[2];
      Jd[3] = 1 + rad + k1 * 2.0 * my + k2 * rho * 4 * my + 6 * p1 * u1 + 2.0 * p2 * u0;
    }
    return true;
  } else if constexpr (MODEL == OKB_DIST_EQUIDISTANT) {
    const double k1 = c.k[0], k2 = c.k[1], k3 = c.k[2], k4 = c.k[3];
    const double r2 = u0 * u0 + u1 * u1;
    const double r = sqrt(r2);
    const double th = atan(r);
    const double th2 = th * th, th4 = th2 * th2, th6 = th4 * th2, th8 = th4 * th4;
    const double poly = 1 + k1 * th2 + k2 * th4 + k3 * th6 + k4 * th8;
    const double thd = th * poly;
    const bool big = r > 1e-8;
    const double scaling = big ? thd / r : 1.0;
    d[0] = scaling * u0; d[1] = scaling * u1;
    if (WANT_J) {
      if (big) {
        // d = s(r) u, s = thd/r:  J = s I + (s'/r) u u^T,  s' = (dthd/dr * r - thd)/r^2,
        // dthd/dr = (poly + th*dpoly/dth) / (1+r^2)   (same function the reference differentiates symbolically)
        const double dpoly = 2 * k1 * th + 4 * k2 * th2 * th + 6 * k3 * th4 * th + 8 * k4 * th6 * th;
        const double dthd = (poly + th * dpoly) / (1.0 + r2);
        const double sp_over_r = (dthd * r - thd) / (r2 * r);
        Jd[0] = scaling + sp_over_r * u0 * u0;
        Jd[1] = sp_over_r * u0 * u1;
        Jd[2] = Jd[1];
        Jd[3] = scaling + sp_over_r * u1 * u1;
      } else {
        Jd[0] = 1; Jd[1] = 0; Jd[2] = 0; Jd[3] = 1;
      }
    }
    return true;
  } else if constexpr (MODEL == OKB_DIST_RADTAN8) {
    const double k1 = c.k[0], k2 = c.k[1], p1 = c.k[2], p2 = c.k[3], k3 = c.k[4], k4 = c.k[5], k5 = c.k[6], k6 = c.k[7];
    const double mx = u0 * u0, my = u1 * u1, mxy = u0 * u1, rho = mx + my;
    if (rho > 9.0) {
      d[0] = d[1] = 0.0;
      if (WANT_J) { Jd[0] = Jd[1] = Jd[2] = Jd[3] = 0.0; }
      return false;
    }
    const double num = 1.0 + ((k3 * rho + k2) * rho + k1) * rho;
    const double den = 1.0 + ((k6 * rho + k5) * rho + k4) * rho;
    const double rad = num / den;
    d[0] = u0 * rad + 2.0 * p1 * mxy + p2 * (rho + 2.0 * mx);
    d[1] = u1 * rad + 2.0 * p2 * mxy + p1 * (rho + 2.0 * my);
    if (WANT_J) {
      // d(rad)/d(rho) = (num' den - num den') / den^2 ; d(rho)/du = 2u
      const double dnum = (3 * k3 * rho + 2 * k2) * rho + k1;
      const double dden = (3 * k6 * rho + 2 * k5) * rho + k4;
      const double drad = (dnum * den - num * dden) / (den * den);
      Jd[0] = rad + 2 * u0 * u0 * drad + 2.0 * p1 * u1 + 6.0 * p2 * u0;
      Jd[1] = 2 * u0 * u1 * drad + 2.0 * p1 * u0 + 2.0 * p2 * u1;
      Jd[2] = Jd[1];
      Jd[3] = rad + 2 * u1 * u1 * drad + 6.0 * p1 * u1 + 2.0 * p2 * u0;
    }
    return true;
  } else {
    static_assert(MODEL == OKB_DIST_NONE, "unknown distortion model");
    d[0] = u0; d[1] = u1;
    if (WANT_J) { Jd[0] = 1; Jd[1] = 0; Jd[2] = 0; Jd[3] = 1; }
    return true;
  }
}

// PinholeCamera::project (+ point Jacobian 2x3 row-major).  Singular depth -> zeros, false.
template <bool WANT_J, int MODEL = kDistAny>
OKB_HD bool project(const CamIntr& c, const double* pt, double* ip, double* J) {
  if (fabs(pt[2]) < 1.0e-12) {
    ip[0] = ip[1] = 0.0;
    if (WANT_J) { J[0] = J[1] = J[2] = J[3] = J[4] = J[5] = 0.0; }
    return false;
  }
  const double rz = 1.0 / pt[2];
  const double u0 = pt[0] * rz, u1 = pt[1] * rz;
  double d[2], Jd[4];
  const bool ok = distort<WANT_J, MODEL>(c, u0, u1, d, Jd);
  if (WANT_J) {
    const double rz2 = rz * rz;
    J[0] = c.fu * Jd[0] * rz;
    J[1] = c.fu * Jd[1] * rz;
    J[2] = -c.fu * (pt[0] * Jd[0] + pt[1] * Jd[1]) * rz2;
    J[3] = c.fv * Jd[2] * rz;
    J[4] = c.fv * Jd[3] * rz;
    J[5] = -c.fv * (pt[0] * Jd[2] + pt[1] * Jd[3]) * rz2;
  }
  ip[0] = c.fu * d[0] + c.cu;
  ip[1] = c.fv * d[1] + c.cv;
  return ok;
}

// ---------------------------------------------------------------- reprojection residual (fused form)
// Camera-from-world transform of one (frame, camera) slot: p_C = R * X_W.xyz + t * X_W.w
struct SlotXf {
  double R[9];   // C_CW = C_CS * C_SW
  double t[3];   // C_CS * (-C_SW t_WS) + (-C_CS t_SC)
};
OKB_HD void make_slot_xf(const double* pose, const double* ext, SlotXf& o) {
  double C_WS[9], C_SC[9];
  q2R(pose + 3, C_WS);
  q2R(ext + 3, C_SC);
  // C_CW = C_SC^T * C_WS^T
  double C_CS[9] = {C_SC[0], C_SC[3], C_SC[6], C_SC[1], C_SC[4], C_SC[7], C_SC[2], C_SC[5], C_SC[8]};
  double C_SW[9] = {C_WS[0], C_WS[3], C_WS[6], C_WS[1], C_WS[4], C_WS[7], C_WS[2], C_WS[5], C_WS[8]};
  mat3mul(C_CS, C_SW, o.R);
  double tSW[3], a[3], b[3];
  mat3vec(C_SW, pose, tSW);           // C_SW t_WS
  mat3vec(C_CS, tSW, a);              // C_CS C_SW t_WS
  mat3vec(C_CS, ext, b);              // C_CS t_SC
  o.t[0] = -a[0] - b[0]; o.t[1] = -a[1] - b[1]; o.t[2] = -a[2] - b[2];
}

// One observation.  Outputs the raw (sqrt-information weighted, NOT robustified) residual r and
// A = sqrtInfo * dproj * C_CW (2x3 row-major; zero if the point is "invalid" exactly as the
// reference zeroes its Jacobians).  Returns hp_C.w (needed by nobody else) via *w_out if non-null.
template <bool WANT_J, int MODEL = kDistAny>
OKB_HD void reproj_slot(const SlotXf& xf, const CamIntr& cam, const double* X /*hom. landmark*/, double z0, double z1,
                        double sqrt_info, double* r, double* A) {
  const double w = X[3];
  double pc[3];
  pc[0] = xf.R[0] * X[0] + xf.R[1] * X[1] + xf.R[2] * X[2] + xf.t[0] * w;
  pc[1] = xf.R[3] * X[0] + xf.R[4] * X[1] + xf.R[5] * X[2] + xf.t[1] * w;
  pc[2] = xf.R[6] * X[0] + xf.R[7] * X[1] + xf.R[8] * X[2] + xf.t[2] * w;
  bool valid = true;
  if (fabs(w) > 1.0e-8) {
    if (pc[2] / w < 0.2) valid = false;
  }
  // projectHomogeneous: w < 0 projects -xyz, Jacobian NOT negated (reference quirk kept)
  double pt[3] = {pc[0], pc[1], pc[2]};
  if (w < 0) { pt[0] = -pt[0]; pt[1] = -pt[1]; pt[2] = -pt[2]; }
  double ip[2], Jp[6];
  project<WANT_J, MODEL>(cam, pt, ip, Jp);
#ifdef __CUDA_ARCH__
  asm volatile("" ::: "memory");      // R is read again below rather than held in registers across the projection
#endif
  r[0] = sqrt_info * (z0 - ip[0]);
  r[1] = sqrt_info * (z1 - ip[1]);
  if (WANT_J) {
    if (valid) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
          A[i * 3 + j] = sqrt_info * (Jp[i * 3] * xf.R[j] + Jp[i * 3 + 1] * xf.R[3 + j] + Jp[i * 3 + 2] * xf.R[6 + j]);
    } else {
#pragma unroll
      for (int i = 0; i < 6; ++i) A[i] = 0.0;
    }
  }
}

// Generic single-block evaluation with all three minimal Jacobians (test hook + extrinsics path):
// J_pose = A [w I, -[p]x], p = X - t_WS w;  J_lm = -A;  J_ext = B [w_S I, -[p_S]x], B = sqrtInfo*dproj*C_CS,
// p_S = hp_S.xyz - t_SC w_S.
OKB_HD void reproj_full(const okb_camera& camera, const double* pose, const double* X, const double* ext, const double* z,
                        double sqrt_info, double* r, double* J0, double* J1, double* J2) {
  CamIntr cam;
  cam_load(camera, cam);
  SlotXf xf;
  make_slot_xf(pose, ext, xf);
  double A[6];
  reproj_slot<true>(xf, cam, X, z[0], z[1], sqrt_info, r, A);
  const double w = X[3];
  const double p[3] = {X[0] - pose[0] * w, X[1] - pose[1] * w, X[2] - pose[2] * w};
  for (int i = 0; i < 2; ++i) {
    const double* a = A + 3 * i;
    if (J0) {
      J0[i * 6 + 0] = w * a[0]; J0[i * 6 + 1] = w * a[1]; J0[i * 6 + 2] = w * a[2];
      // -a^T [p]x = (p x a)^T
      J0[i * 6 + 3] = p[1] * a[2] - p[2] * a[1];
      J0[i * 6 + 4] = p[2] * a[0] - p[0] * a[2];
      J0[i * 6 + 5] = p[0] * a[1] - p[1] * a[0];
    }
    if (J1) { J1[i * 3 + 0] = -a[0]; J1[i * 3 + 1] = -a[1]; J1[i * 3 + 2] = -a[2]; }
  }
  if (J2) {
    // B = A * C_WS ... (A = B C_SW  =>  B = A C_SW^T = A C_WS)
    double C_WS[9];
    q2R(pose + 3, C_WS);
    double C_SW[9] = {C_WS[0], C_WS[3], C_WS[6], C_WS[1], C_WS[4], C_WS[7], C_WS[2], C_WS[5], C_WS[8]};
    double hpS[3], tmp[3] = {p[0], p[1], p[2]};
    mat3vec(C_SW, tmp, hpS);  // hp_S.xyz = C_SW (X - t w)
    const double pS[3] = {hpS[0] - ext[0] * w, hpS[1] - ext[1] * w, hpS[2] - ext[2] * w};
    for (int i = 0; i < 2; ++i) {
      double b[3];
      // b = a^T C_WS  (row vector times matrix)
      b[0] = A[3 * i] * C_WS[0] + A[3 * i + 1] * C_WS[3] + A[3 * i + 2] * C_WS[6];
      b[1] = A[3 * i] * C_WS[1] + A[3 * i + 1] * C_WS[4] + A[3 * i + 2] * C_WS[7];
      b[2] = A[3 * i] * C_WS[2] + A[3 * i + 1] * C_WS[5] + A[3 * i + 2] * C_WS[8];
      J2[i * 6 + 0] = w * b[0]; J2[i * 6 + 1] = w * b[1]; J2[i * 6 + 2] = w * b[2];
      J2[i * 6 + 3] = pS[1] * b[2] - pS[2] * b[1];
      J2[i * 6 + 4] = pS[2] * b[0] - pS[0] * b[2];
      J2[i * 6 + 5] = pS[0] * b[1] - pS[1] * b[0];
    }
  }
}

// ---------------------------------------------------------------- priors
// e = [t_m - t; 2 vec(q_m * q^-1)],  J_min = sqrtInfo * [-I 0; 0 -plus(q_dp)_3x3]   (PoseError.cpp:86-136)
OKB_HD void pose_error_e(const double* meas, const double* pose, double* e, double* Jrot /*3x3 = plus(dq) block*/) {
  double qm[4] = {meas[3], meas[4], meas[5], meas[6]}, q[4] = {pose[3], pose[4], pose[5], pose[6]};
  qnormalize(qm); qnormalize(q);
  double qi[4], dq[4];
  qinv(q, qi);
  qmul(qm, qi, dq);
  qnormalize(dq);
  e[0] = meas[0] - pose[0]; e[1] = meas[1] - pose[1]; e[2] = meas[2] - pose[2];
  e[3] = 2 * dq[0]; e[4] = 2 * dq[1]; e[5] = 2 * dq[2];
  if (Jrot) {
    Jrot[0] = dq[3];  Jrot[1] = -dq[2]; Jrot[2] = dq[1];
    Jrot[3] = dq[2];  Jrot[4] = dq[3];  Jrot[5] = -dq[0];
    Jrot[6] = -dq[1]; Jrot[7] = dq[0];  Jrot[8] = dq[3];
  }
}
// Full PoseError: r = S e, J = S * Jmin (6x6 row-major)
OKB_HD void pose_error(const double* meas, const double* S, const double* pose, double* r, double* J) {
  double e[6], Q[9];
  pose_error_e(meas, pose, e, Q);
  for (int i = 0; i < 6; ++i) {
    double s = 0;
    for (int k = 0; k < 6; ++k) s += S[i * 6 + k] * e[k];
    r[i] = s;
  }
  if (J) {
    for (int i = 0; i < 6; ++i) {
      for (int j = 0; j < 3; ++j) J[i * 6 + j] = -S[i * 6 + j];
      for (int j = 0; j < 3; ++j)
        J[i * 6 + 3 + j] = -(S[i * 6 + 3] * Q[j] + S[i * 6 + 4] * Q[3 + j] + S[i * 6 + 5] * Q[6 + j]);
    }
  }
}
// RelativePoseError (RelativePoseError.cpp:84-162)
OKB_HD void relative_pose_error(const double* S, const double* p0, const double* p1, double* r, double* J0, double* J1) {
  double q0[4] = {p0[3], p0[4], p0[5], p0[6]}, q1[4] = {p1[3], p1[4], p1[5], p1[6]};
  qnormalize(q0); qnormalize(q1);
  double qi[4], dq[4];
  qinv(q0, qi);
  qmul(q1, qi, dq);
  qnormalize(dq);
  const double e[6] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2], 2 * dq[0], 2 * dq[1], 2 * dq[2]};
  for (int i = 0; i < 6; ++i) {
    double s = 0;
    for (int k = 0; k < 6; ++k) s += S[i * 6 + k] * e[k];
    r[i] = s;
  }
  const double P[9] = {dq[3], -dq[2], dq[1], dq[2], dq[3], -dq[0], -dq[1], dq[0], dq[3]};   // plus(dq) 3x3
  const double O[9] = {dq[3], dq[2], -dq[1], -dq[2], dq[3], dq[0], dq[1], -dq[0], dq[3]};   // oplus(dq) 3x3
  for (int i = 0; i < 6; ++i) {
    for (int j = 0; j < 3; ++j) {
      if (J0) J0[i * 6 + j] = -S[i * 6 + j];
      if (J1) J1[i * 6 + j] = S[i * 6 + j];
    }
    for (int j = 0; j < 3; ++j) {
      if (J0) J0[i * 6 + 3 + j] = -(S[i * 6 + 3] * P[j] + S[i * 6 + 4] * P[3 + j] + S[i * 6 + 5] * P[6 + j]);
      if (J1) J1[i * 6 + 3 + j] = (S[i * 6 + 3] * O[j] + S[i * 6 + 4] * O[3 + j] + S[i * 6 + 5] * O[6 + j]);
    }
  }
}
// The 3x3 block (lift(x0) * plus(x))_rot = oplus(q * q0^-1)[0:3,0:3] used by the marginalisation prior
OKB_HD void marg_pose_rot_block(const double* x0, const double* x, double* B) {
  double q[4] = {x[3], x[4], x[5], x[6]};
  qnormalize(q);
  // lift uses the raw x0 quaternion conjugate (PoseLocalParameterization.cpp:133-147): q_inv = conj(x0)
  const double qc[4] = {-x0[3], -x0[4], -x0[5], x0[6]};
  double d[4];
  qmul(q, qc, d);
  B[0] = d[3];  B[1] = d[2];  B[2] = -d[1];
  B[3] = -d[2]; B[4] = d[3];  B[5] = d[0];
  B[6] = d[1];  B[7] = -d[0]; B[8] = d[3];
}

}  // namespace okb
