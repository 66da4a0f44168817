// Epipolar geometry in float64: patch->image affine, two-view triangulation
// (homogeneous DLT / linear LS / iterative LS) and projection to labels.
// Reference arithmetic: lib/utils/triangulation.py, lib/utils/img_utils.py:63-111,
// 141-155,193-243, lib/utils/prep_h36m.py:170-204, lib/core/integral_loss.py:170-205.
// The SVDs the reference obtains from OpenCV (cv2.triangulatePoints,
// cv2.solve(DECOMP_SVD)) are one-sided Jacobi SVDs on the un-squared matrix,
// as in OpenCV's JacobiSVD (so the condition number is not squared).
//
// One thread per (pair, joint): the problem is a few hundred bytes per joint
// and latency-bound at real sizes (64 pairs x 17 joints); no tensor cores.
// Compiled with --fmad=false so that a*b+c rounds twice as on the CPU.
#include "common.cuh"
#include "camera.cuh"
#include <float.h>

namespace {

// One-sided (Hestenes) Jacobi: rotate columns of A (R x C) until mutually
// orthogonal; V (C x C) accumulates the right rotations.  On exit
// A = U*diag(sigma) (columns), sigma_j = ||A[:,j]||.
template <int R, int C>
__host__ __device__ void jacobi_onesided(double (&A)[R][C], double (&V)[C][C]) {
#pragma unroll
  for (int i = 0; i < C; ++i)
#pragma unroll
    for (int j = 0; j < C; ++j) V[i][j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 30; ++sweep) {
    bool changed = false;
#pragma unroll
    for (int p = 0; p < C - 1; ++p) {
#pragma unroll
      for (int q = p + 1; q < C; ++q) {
        double a = 0, b = 0, g = 0;
#pragma unroll
        for (int i = 0; i < R; ++i) {
          a += A[i][p] * A[i][p];
          b += A[i][q] * A[i][q];
          g += A[i][p] * A[i][q];
        }
        if (fabs(g) <= DBL_EPSILON * sqrt(a * b) || g == 0.0) continue;
        changed = true;
        const double zeta = (b - a) / (2.0 * g);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const double x = A[i][p], y = A[i][q];
          A[i][p] = c * x - s * y;
          A[i][q] = s * x + c * y;
        }
#pragma unroll
        for (int i = 0; i < C; ++i) {
          const double x = V[i][p], y = V[i][q];
          V[i][p] = c * x - s * y;
          V[i][q] = s * x + c * y;
        }
      }
    }
    if (!changed) break;
  }
}

// least-squares solve of A(4x3) x = b via SVD, as cv2.solve(.., DECOMP_SVD)
__device__ void solve_ls_4x3(const double (&A0)[4][3], const double (&b)[4], double (&x)[3]) {
  double A[4][3], V[3][3];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) A[i][j] = A0[i][j];
  jacobi_onesided<4, 3>(A, V);
  double s2[3], y[3], ssum = 0;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    double n2 = 0, d = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) { n2 += A[i][j] * A[i][j]; d += A[i][j] * b[i]; }
    s2[j] = n2;
    y[j] = d;
    ssum += sqrt(n2);
  }
  const double thr = DBL_EPSILON * 2.0 * ssum;  // cv::SVD::backSubst threshold
#pragma unroll
  for (int j = 0; j < 3; ++j) y[j] = (sqrt(s2[j]) > thr) ? y[j] / s2[j] : 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) x[i] = V[i][0] * y[0] + V[i][1] * y[1] + V[i][2] * y[2];
}

// triangulation.py:139-150 / :80-92: rows C*P[:3,:3], b = -(C*P[:3,3]),
// C = [[-1,0,u],[0,-1,v]]
__device__ void build_Ab(const double* u1, const double* P1, const double* u2, const double* P2,
                         double (&A)[4][3], double (&b)[4]) {
#pragma unroll
  for (int v = 0; v < 2; ++v) {
    const double* u = v ? u2 : u1;
    const double* P = v ? P2 : P1;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      A[2 * v + 0][k] = -P[0 * 4 + k] + u[0] * P[2 * 4 + k];
      A[2 * v + 1][k] = -P[1 * 4 + k] + u[1] * P[2 * 4 + k];
    }
    b[2 * v + 0] = -(-P[0 * 4 + 3] + u[0] * P[2 * 4 + 3]);
    b[2 * v + 1] = -(-P[1 * 4 + 3] + u[1] * P[2 * 4 + 3]);
  }
}

// --------------------------------------------------------------- polynomial (optimal) correction
// lib/utils/triangulation.py:184-220: F from the two projection matrices, cv2.correctMatches
// (Hartley-Sturm, Hartley & Zisserman Alg. 12.1) and the homogeneous DLT on the corrected
// matches.  OpenCV finds the six roots of the stationarity polynomial with cvSolvePoly; here:
// Laguerre iterations with deflation and a polishing pass on the un-deflated polynomial
// (complex float64), which reaches the same roots to rounding.
struct cplx { double re, im; };
__host__ __device__ inline cplx cmk(double r, double i) { cplx c; c.re = r; c.im = i; return c; }
__host__ __device__ inline cplx cadd(cplx a, cplx b) { return cmk(a.re + b.re, a.im + b.im); }
__host__ __device__ inline cplx csub(cplx a, cplx b) { return cmk(a.re - b.re, a.im - b.im); }
__host__ __device__ inline cplx cmul(cplx a, cplx b) {
  return cmk(a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re);
}
__host__ __device__ inline cplx cscale(cplx a, double k) { return cmk(a.re * k, a.im * k); }
__host__ __device__ inline double cabs2(cplx a) { return hypot(a.re, a.im); }
__host__ __device__ inline cplx cdiv(cplx a, cplx b) {       // Smith's algorithm
  if (fabs(b.re) >= fabs(b.im)) {
    const double r = b.im / b.re, den = b.re + r * b.im;
    return cmk((a.re + r * a.im) / den, (a.im - r * a.re) / den);
  }
  const double r = b.re / b.im, den = b.im + r * b.re;
  return cmk((a.re * r + a.im) / den, (a.im * r - a.re) / den);
}
__host__ __device__ inline cplx csqrt2(cplx z) {
  if (z.re == 0.0 && z.im == 0.0) return cmk(0.0, 0.0);
  const double x = fabs(z.re), y = fabs(z.im);
  double w;
  if (x >= y) { const double r = y / x; w = sqrt(x) * sqrt(0.5 * (1.0 + sqrt(1.0 + r * r))); }
  else { const double r = x / y; w = sqrt(y) * sqrt(0.5 * (r + sqrt(1.0 + r * r))); }
  if (z.re >= 0.0) return cmk(w, z.im / (2.0 * w));
  return cmk(y / (2.0 * w), z.im >= 0.0 ? w : -w);
}

// one root of sum_{k<=m} a[k] x^k by Laguerre's method, starting from (and returned in) x
__host__ __device__ inline void laguerre(const cplx* a, int m, cplx& x) {
  const double frac[9] = {0.0, 0.5, 0.25, 0.75, 0.13, 0.38, 0.62, 0.88, 1.0};
  for (int iter = 1; iter <= 80; ++iter) {
    cplx b = a[m], d = cmk(0, 0), f = cmk(0, 0);
    double err = cabs2(b);
    const double abx = cabs2(x);
    for (int j = m - 1; j >= 0; --j) {
      f = cadd(cmul(x, f), d);
      d = cadd(cmul(x, d), b);
      b = cadd(cmul(x, b), a[j]);
      err = cabs2(b) + abx * err;
    }
    if (cabs2(b) <= err * 2.0e-16) return;                 // on the root to rounding
    const cplx g = cdiv(d, b), g2 = cmul(g, g);
    const cplx h = csub(g2, cscale(cdiv(f, b), 2.0));
    const cplx sq = csqrt2(cscale(csub(cscale(h, (double)m), g2), (double)(m - 1)));
    cplx gp = cadd(g, sq);
    const cplx gm = csub(g, sq);
    const double abp = cabs2(gp), abm = cabs2(gm);
    if (abp < abm) gp = gm;
    cplx dx;
    if (fmax(abp, abm) > 0.0) dx = cdiv(cmk((double)m, 0.0), gp);
    else dx = cscale(cmk(cos((double)iter), sin((double)iter)), 1.0 + abx);
    const cplx x1 = csub(x, dx);
    if (x.re == x1.re && x.im == x1.im) return;
    if (iter % 10) x = x1;
    else x = csub(x, cscale(dx, frac[(iter / 10) % 9]));
  }
}

// real parts of the roots of the real polynomial sum_{k<=6} k[k] t^k (leading zeros stripped)
__host__ __device__ inline int poly6_root_reals(const double* k, double* re) {
  int m = 6;
  double big = 0.0;
  for (int i = 0; i <= 6; ++i) big = fmax(big, fabs(k[i]));
  while (m > 0 && fabs(k[m]) <= big * 1e-300) --m;
  if (m == 0) return 0;
  cplx a[7], ad[7];
  for (int i = 0; i <= m; ++i) { a[i] = cmk(k[i], 0.0); ad[i] = a[i]; }
  cplx roots[6];
  for (int j = m; j >= 1; --j) {
    cplx x = cmk(0.0, 0.0);
    laguerre(ad, j, x);
    if (fabs(x.im) <= 4.0e-16 * fabs(x.re)) x.im = 0.0;
    roots[j - 1] = x;
    cplx b = ad[j];
    for (int jj = j - 1; jj >= 0; --jj) {                  // forward deflation
      const cplx c = ad[jj];
      ad[jj] = b;
      b = cadd(cmul(x, b), c);
    }
  }
  for (int j = 0; j < m; ++j) {
    laguerre(a, m, roots[j]);                              // polish on the full polynomial
    re[j] = roots[j].re;
  }
  return m;
}

// [t]x R of the canonical pair P2_full * inv(P1_full)  (triangulation.py:198-204)
__host__ __device__ inline void fundamental_from_P(const double* P1, const double* P2, double* F) {
  // inv([M p; 0 1]) = [M^-1  -M^-1 p; 0 1]
  const double m00 = P1[0], m01 = P1[1], m02 = P1[2], m10 = P1[4], m11 = P1[5], m12 = P1[6],
               m20 = P1[8], m21 = P1[9], m22 = P1[10];
  const double c00 = m11 * m22 - m12 * m21, c01 = m12 * m20 - m10 * m22, c02 = m10 * m21 - m11 * m20;
  const double det = m00 * c00 + m01 * c01 + m02 * c02;
  double Mi[3][3];
  Mi[0][0] = c00 / det; Mi[0][1] = (m02 * m21 - m01 * m22) / det; Mi[0][2] = (m01 * m12 - m02 * m11) / det;
  Mi[1][0] = c01 / det; Mi[1][1] = (m00 * m22 - m02 * m20) / det; Mi[1][2] = (m02 * m10 - m00 * m12) / det;
  Mi[2][0] = c02 / det; Mi[2][1] = (m01 * m20 - m00 * m21) / det; Mi[2][2] = (m00 * m11 - m01 * m10) / det;
  double R[3][3], t[3];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c)
      R[r][c] = P2[r * 4 + 0] * Mi[0][c] + P2[r * 4 + 1] * Mi[1][c] + P2[r * 4 + 2] * Mi[2][c];
    t[r] = P2[r * 4 + 3] - (R[r][0] * P1[3] + R[r][1] * P1[7] + R[r][2] * P1[11]);
    // a translation that is pure cancellation noise (identical camera centres) is exactly zero:
    // the reference's F is then the zero matrix and its correction all-NaN (:213-217)
    const double mag = fabs(P2[r * 4 + 3]) + fabs(R[r][0] * P1[3]) + fabs(R[r][1] * P1[7]) +
                       fabs(R[r][2] * P1[11]);
    if (fabs(t[r]) <= 64.0 * DBL_EPSILON * mag) t[r] = 0.0;
  }
  for (int c = 0; c < 3; ++c) {                            // F[:,c] = t x R[:,c]
    F[0 * 3 + c] = t[1] * R[2][c] - t[2] * R[1][c];
    F[1 * 3 + c] = t[2] * R[0][c] - t[0] * R[2][c];
    F[2 * 3 + c] = t[0] * R[1][c] - t[1] * R[0][c];
  }
}

// cv2.correctMatches for one match (u1, u2 updated in place)
__host__ __device__ inline void correct_match(const double* F, double* u1, double* u2) {
  const double x1 = u1[0], y1 = u1[1], x2 = u2[0], y2 = u2[1];
  // TFT = T2i^T F T1i with T = [1 0 x; 0 1 y; 0 0 1]
  double G[3][3];
  for (int r = 0; r < 3; ++r) {
    G[r][0] = F[r * 3 + 0];
    G[r][1] = F[r * 3 + 1];
    G[r][2] = F[r * 3 + 0] * x1 + F[r * 3 + 1] * y1 + F[r * 3 + 2];
  }
  double T[3][3];
  for (int c = 0; c < 3; ++c) {
    T[0][c] = G[0][c];
    T[1][c] = G[1][c];
    T[2][c] = x2 * G[0][c] + y2 * G[1][c] + G[2][c];
  }
  // epipoles: right null vector = cross product of the two most independent rows, left null
  // vector likewise from the columns (OpenCV takes them from the SVD of the rank-2 matrix)
  auto null_of = [&](bool rows, double (&e)[3]) {
    double best = -1.0;
    for (int i = 0; i < 3; ++i) {
      const int j = (i + 1) % 3;
      double a[3], b[3], c[3];
      for (int k = 0; k < 3; ++k) { a[k] = rows ? T[i][k] : T[k][i]; b[k] = rows ? T[j][k] : T[k][j]; }
      c[0] = a[1] * b[2] - a[2] * b[1];
      c[1] = a[2] * b[0] - a[0] * b[2];
      c[2] = a[0] * b[1] - a[1] * b[0];
      const double n = c[0] * c[0] + c[1] * c[1] + c[2] * c[2];
      if (n > best) { best = n; e[0] = c[0]; e[1] = c[1]; e[2] = c[2]; }
    }
    const double s = sqrt(e[0] * e[0] + e[1] * e[1]);
    e[0] /= s; e[1] /= s; e[2] /= s;
  };
  double e1[3], e2[3];
  null_of(true, e1);
  null_of(false, e2);
  // RF = R2 TFT R1^T, R = [ex ey 0; -ey ex 0; 0 0 1]
  double H[3][3];
  for (int r = 0; r < 3; ++r) {                            // H = TFT R1^T
    H[r][0] = T[r][0] * e1[0] + T[r][1] * e1[1];
    H[r][1] = -T[r][0] * e1[1] + T[r][1] * e1[0];
    H[r][2] = T[r][2];
  }
  const double a = -e2[1] * H[0][1] + e2[0] * H[1][1], b = -e2[1] * H[0][2] + e2[0] * H[1][2];
  const double c = H[2][1], d = H[2][2];
  const double f1 = e1[2], f2 = e2[2];
  // g(t) = t((at+b)^2 + f2^2(ct+d)^2)^2 - (ad-bc)(1+f1^2 t^2)^2 (at+b)(ct+d), ascending powers
  const double q0 = b * b + f2 * f2 * d * d, q1 = 2.0 * (a * b + f2 * f2 * c * d),
               q2 = a * a + f2 * f2 * c * c;
  const double qq[5] = {q0 * q0, 2.0 * q0 * q1, 2.0 * q0 * q2 + q1 * q1, 2.0 * q1 * q2, q2 * q2};
  const double w = a * d - b * c, ff = f1 * f1;
  const double r0 = b * d, r1 = a * d + b * c, r2 = a * c;              // (at+b)(ct+d)
  const double p4[5] = {1.0, 0.0, 2.0 * ff, 0.0, ff * ff};               // (1+f1^2 t^2)^2
  double k[7] = {0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 5; ++i) k[i + 1] += qq[i];
  for (int i = 0; i < 5; ++i) {
    k[i] -= w * p4[i] * r0;
    k[i + 1] -= w * p4[i] * r1;
    k[i + 2] -= w * p4[i] * r2;
  }
  double re[6];
  const int nr = poly6_root_reals(k, re);
  double smin = DBL_MAX, tmin = 0.0;
  for (int i = 0; i < nr; ++i) {
    const double t = re[i];
    const double n1 = c * t + d, n0 = a * t + b;
    const double sv = t * t / (1.0 + ff * t * t) + n1 * n1 / (n0 * n0 + f2 * f2 * n1 * n1);
    if (sv < smin) { smin = sv; tmin = t; }
  }
  const double sinf = 1.0 / ff + c * c / (a * a + f2 * f2 * c * c);
  double l1[3], l2[3];
  if (sinf < smin) {                                       // minimum at t = infinity
    l1[0] = f1; l1[1] = 0.0; l1[2] = -1.0;
    l2[0] = -f2 * c; l2[1] = a; l2[2] = c;
  } else {
    l1[0] = tmin * f1; l1[1] = 1.0; l1[2] = -tmin;
    l2[0] = -f2 * (c * tmin + d); l2[1] = a * tmin + b; l2[2] = c * tmin + d;
  }
  // closest points to the origin on the two lines, rotated and translated back
  const double h1[3] = {-l1[0] * l1[2], -l1[1] * l1[2], l1[0] * l1[0] + l1[1] * l1[1]};
  const double h2[3] = {-l2[0] * l2[2], -l2[1] * l2[2], l2[0] * l2[0] + l2[1] * l2[1]};
  const double g1[3] = {e1[0] * h1[0] - e1[1] * h1[1], e1[1] * h1[0] + e1[0] * h1[1], h1[2]};   // R1^T h1
  const double g2[3] = {e2[0] * h2[0] - e2[1] * h2[1], e2[1] * h2[0] + e2[0] * h2[1], h2[2]};
  u1[0] = (g1[0] + x1 * g1[2]) / g1[2];
  u1[1] = (g1[1] + y1 * g1[2]) / g1[2];
  u2[0] = (g2[0] + x2 * g2[2]) / g2[2];
  u2[1] = (g2[1] + y2 * g2[2]) / g2[2];
}

// cv2.findFundamentalMat(u1, u2, FM_8POINT) for one pair (OpenCV calib3d fundam.cpp run8Point):
// points rounded to float32 (findFundamentalMat converts its inputs to CV_32F), isotropic
// normalisation (centroid, mean distance sqrt 2), the 9x9 normal matrix A^T A, its eigenvector of
// the smallest eigenvalue, rank-2 projection through the SVD of the 3x3, de-normalisation,
// F[2][2] = 1.  Returns false where OpenCV returns no matrix (degenerate point sets).
__host__ __device__ inline bool fundamental_8point(const double* u1, const double* u2, int stride_u,
                                                   int J, double* F) {
  double c1[2] = {0, 0}, c2[2] = {0, 0};
  for (int i = 0; i < J; ++i) {
    c1[0] += (double)(float)u1[(int64_t)i * stride_u];
    c1[1] += (double)(float)u1[(int64_t)i * stride_u + 1];
    c2[0] += (double)(float)u2[(int64_t)i * stride_u];
    c2[1] += (double)(float)u2[(int64_t)i * stride_u + 1];
  }
  const double t = 1.0 / J;
  c1[0] *= t; c1[1] *= t; c2[0] *= t; c2[1] *= t;
  double s1 = 0, s2 = 0;
  for (int i = 0; i < J; ++i) {
    const double x1 = (double)(float)u1[(int64_t)i * stride_u] - c1[0];
    const double y1 = (double)(float)u1[(int64_t)i * stride_u + 1] - c1[1];
    const double x2 = (double)(float)u2[(int64_t)i * stride_u] - c2[0];
    const double y2 = (double)(float)u2[(int64_t)i * stride_u + 1] - c2[1];
    s1 += sqrt(x1 * x1 + y1 * y1);
    s2 += sqrt(x2 * x2 + y2 * y2);
  }
  s1 *= t; s2 *= t;
  if (s1 < 1.1920929e-07 || s2 < 1.1920929e-07) return false;     // FLT_EPSILON
  s1 = sqrt(2.0) / s1;
  s2 = sqrt(2.0) / s2;
  double G[9][9], V[9][9];
  for (int a = 0; a < 9; ++a)
    for (int b = 0; b < 9; ++b) G[a][b] = 0.0;
  for (int i = 0; i < J; ++i) {
    const double x1 = ((double)(float)u1[(int64_t)i * stride_u] - c1[0]) * s1;
    const double y1 = ((double)(float)u1[(int64_t)i * stride_u + 1] - c1[1]) * s1;
    const double x2 = ((double)(float)u2[(int64_t)i * stride_u] - c2[0]) * s2;
    const double y2 = ((double)(float)u2[(int64_t)i * stride_u + 1] - c2[1]) * s2;
    const double r[9] = {x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1.0};
    for (int a = 0; a < 9; ++a)
      for (int b = 0; b < 9; ++b) G[a][b] += r[a] * r[b];
  }
  // eigenvectors of the symmetric PSD normal matrix = its right singular vectors
  jacobi_onesided<9, 9>(G, V);
  int best = 0, nz = 0;
  double bn = DBL_MAX;
  for (int j = 0; j < 9; ++j) {
    double n2 = 0;
    for (int i = 0; i < 9; ++i) n2 += G[i][j] * G[i][j];
    if (sqrt(n2) >= DBL_EPSILON) ++nz;
    if (n2 < bn) { bn = n2; best = j; }
  }
  if (nz < 8) return false;                         // OpenCV: fewer than 8 non-zero eigenvalues
  double F0[3][3], W[3][3];
  for (int i = 0; i < 9; ++i) {
    double v = V[i][0];
    for (int j = 1; j < 9; ++j)
      if (best == j) v = V[i][j];
    F0[i / 3][i % 3] = v;
  }
  // rank 2: drop the smallest singular value
  double A[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) A[i][j] = F0[i][j];
  jacobi_onesided<3, 3>(A, W);                      // A = U diag(sigma) (columns), F0 = A W^T
  int sm = 0;
  double sn = DBL_MAX;
  for (int j = 0; j < 3; ++j) {
    const double n2 = A[0][j] * A[0][j] + A[1][j] * A[1][j] + A[2][j] * A[2][j];
    if (n2 < sn) { sn = n2; sm = j; }
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double v = 0;
      for (int k = 0; k < 3; ++k)
        if (k != sm) v += A[i][k] * W[j][k];
      F0[i][j] = v;
    }
  // F = T2^T F0 T1, T = [s 0 -s*cx; 0 s -s*cy; 0 0 1]
  const double T1[3][3] = {{s1, 0, -s1 * c1[0]}, {0, s1, -s1 * c1[1]}, {0, 0, 1}};
  const double T2[3][3] = {{s2, 0, -s2 * c2[0]}, {0, s2, -s2 * c2[1]}, {0, 0, 1}};
  double M[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double v = 0;
      for (int k = 0; k < 3; ++k) v += F0[i][k] * T1[k][j];
      M[i][j] = v;
    }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double v = 0;
      for (int k = 0; k < 3; ++k) v += T2[k][i] * M[k][j];
      F[i * 3 + j] = v;
    }
  if (fabs(F[8]) > 1.1920929e-07) {
    const double inv = 1.0 / F[8];
    for (int k = 0; k < 9; ++k) F[k] *= inv;
  }
  return true;
}

// Fundamental matrix per pair for the polynomial method (triangulation.py:198-217): from the
// projection matrices; when the optimal correction with it is NaN for EVERY joint of the pair
// (identical / degenerate cameras) -- or always, for mode 4 -- the 8-point estimate from the
// matches themselves, as the reference falls back to.  One thread per pair.
__global__ void pair_fundamental_kernel(const double* __restrict__ u1, const double* __restrict__ u2,
                                        int stride_u, const double* __restrict__ P1,
                                        const double* __restrict__ P2, int NP, int J, int method,
                                        double* __restrict__ Fout) {
  const int pair = blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= NP) return;
  double F[9];
  fundamental_from_P(P1 + pair * 12, P2 + pair * 12, F);
  bool fallback = method == 4;
  if (!fallback) {
    bool all1 = true, all2 = true;
    for (int j = 0; j < J && (all1 || all2); ++j) {
      const int64_t o = ((int64_t)pair * J + j) * stride_u;
      double a1[2] = {u1[o], u1[o + 1]}, a2[2] = {u2[o], u2[o + 1]};
      correct_match(F, a1, a2);
      if (!(isnan(a1[0]) && isnan(a1[1]))) all1 = false;
      if (!(isnan(a2[0]) && isnan(a2[1]))) all2 = false;
    }
    fallback = all1 || all2;
  }
  if (fallback) {
    double F8[9];
    if (fundamental_8point(u1 + (int64_t)pair * J * stride_u, u2 + (int64_t)pair * J * stride_u,
                           stride_u, J, F8))
      for (int k = 0; k < 9; ++k) F[k] = F8[k];
  }
  for (int k = 0; k < 9; ++k) Fout[pair * 9 + k] = F[k];
}

__global__ void triangulate_kernel(const double* __restrict__ u1, const double* __restrict__ u2,
                                   int stride_u, const double* __restrict__ P1,
                                   const double* __restrict__ P2, int NP, int J, int method,
                                   double tol, const double* __restrict__ Fpair,
                                   double* __restrict__ X, int32_t* __restrict__ status) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= NP * J) return;
  const int pair = idx / J;
  double p1[12], p2[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) { p1[k] = P1[pair * 12 + k]; p2[k] = P2[pair * 12 + k]; }
  double a1[2] = {u1[(int64_t)idx * stride_u], u1[(int64_t)idx * stride_u + 1]};
  double a2[2] = {u2[(int64_t)idx * stride_u], u2[(int64_t)idx * stride_u + 1]};
  double x[3];
  int st;
  if (method >= 3) {   // triangulation.py:184-220: optimal correction, then the homogeneous DLT
    double F[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) F[k] = Fpair[pair * 9 + k];
    correct_match(F, a1, a2);
  }
  if (method == 0 || method >= 3) {
    // triangulation.py:22 cv2.triangulatePoints: A rows x*P[2]-P[0], y*P[2]-P[1]
    double A[4][4], V[4][4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      A[0][k] = a1[0] * p1[8 + k] - p1[0 + k];
      A[1][k] = a1[1] * p1[8 + k] - p1[4 + k];
      A[2][k] = a2[0] * p2[8 + k] - p2[0 + k];
      A[3][k] = a2[1] * p2[8 + k] - p2[4 + k];
    }
    jacobi_onesided<4, 4>(A, V);
    int best = 0;
    double bn = DBL_MAX;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double n2 = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) n2 += A[i][j] * A[i][j];
      if (n2 < bn) { bn = n2; best = j; }
    }
    double h[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      h[i] = V[i][0];
#pragma unroll
      for (int j = 1; j < 4; ++j)
        if (best == j) h[i] = V[i][j];
    }
    x[0] = h[0] / h[3]; x[1] = h[1] / h[3]; x[2] = h[2] / h[3];  // :24
    const double mx = fmax(fabs(x[0]), fmax(fabs(x[1]), fabs(x[2])));
    st = (mx <= 1.e16) ? 1 : 0;  // :25 (NaN compares false)
  } else {
    double A[4][3], b[4];
    build_Ab(a1, p1, a2, p2, A, b);
    if (method == 1) {
      solve_ls_4x3(A, b, x);
      st = 1;
    } else {
      double d1 = 1.0, d2 = 1.0, d1n = 1.0, d2n = 1.0;
      for (int it = 0; it < 10; ++it) {   // :152
        solve_ls_4x3(A, b, x);
        d1n = ((p1[8] * x[0] + p1[9] * x[1]) + p1[10] * x[2]) + p1[11];   // :158
        d2n = ((p2[8] * x[0] + p2[9] * x[1]) + p2[10] * x[2]) + p2[11];
        if (fabs(d1n - d1) <= tol && fabs(d2n - d2) <= tol) break;  // :161-163
        const double r1 = 1.0 / d1n, r2 = 1.0 / d2n;
        // :165-169 CUMULATIVE re-weighting of the already weighted rows
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          A[0][k] *= r1; A[1][k] *= r1; A[2][k] *= r2; A[3][k] *= r2;
        }
        b[0] *= r1; b[1] *= r1; b[2] *= r2; b[3] *= r2;
        d1 = d1n; d2 = d2n;
      }
      st = (d1n > 0 && d2n > 0) ? 1 : 0;  // :175-176 (i < 10 always holds)
      if (d1n <= 0) st -= 1;
      if (d2n <= 0) st -= 2;
    }
  }
  X[(int64_t)idx * 3 + 0] = x[0];
  X[(int64_t)idx * 3 + 1] = x[1];
  X[(int64_t)idx * 3 + 2] = x[2];
  if (status) status[idx] = st;
}

// --------------------------------------------------------------- N-view homogeneous DLT
// SURVEY 8(f) row 3: the V-view generalisation of triangulation.py:8-27 (not in the reference,
// which only pairs two views): A (2V x 4) rows u*P[2]-P[0], v*P[2]-P[1] per view, X = right
// singular vector of the smallest singular value, de-homogenised.  V <= 4 (one tuple).
template <int V>
__host__ __device__ inline int dlt_nview(const double* u /*[V][2]*/, const double* P /*[V][12]*/,
                                         double* x /*[3]*/) {
  double A[2 * V][4], Vm[4][4];
  for (int v = 0; v < V; ++v)
    for (int k = 0; k < 4; ++k) {
      A[2 * v + 0][k] = u[v * 2 + 0] * P[v * 12 + 8 + k] - P[v * 12 + 0 + k];
      A[2 * v + 1][k] = u[v * 2 + 1] * P[v * 12 + 8 + k] - P[v * 12 + 4 + k];
    }
  jacobi_onesided<2 * V, 4>(A, Vm);
  int best = 0;
  double bn = DBL_MAX;
  for (int j = 0; j < 4; ++j) {
    double n2 = 0;
    for (int i = 0; i < 2 * V; ++i) n2 += A[i][j] * A[i][j];
    if (n2 < bn) { bn = n2; best = j; }
  }
  double h[4];
  for (int i = 0; i < 4; ++i) h[i] = Vm[i][best];
  x[0] = h[0] / h[3]; x[1] = h[1] / h[3]; x[2] = h[2] / h[3];
  const double mx = fmax(fabs(x[0]), fmax(fabs(x[1]), fabs(x[2])));
  return (mx <= 1.e16) ? 1 : 0;
}

// u [NT][V][J][stride_u], P [NT][V][12] -> X [NT][J][3], status [NT][J]; one thread per (tuple, joint)
__global__ void triangulate_nview_kernel(const double* __restrict__ u, int stride_u,
                                         const double* __restrict__ P, int NT, int V, int J,
                                         double* __restrict__ X, int32_t* __restrict__ status) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= NT * J) return;
  const int t = idx / J, j = idx - t * J;
  double uu[8], pp[48], x[3];
  for (int v = 0; v < V; ++v) {
    const double* up = u + (((int64_t)t * V + v) * J + j) * stride_u;
    uu[v * 2 + 0] = up[0];
    uu[v * 2 + 1] = up[1];
    for (int k = 0; k < 12; ++k) pp[v * 12 + k] = P[((int64_t)t * V + v) * 12 + k];
  }
  int st;
  if (V == 2) st = dlt_nview<2>(uu, pp, x);
  else if (V == 3) st = dlt_nview<3>(uu, pp, x);
  else st = dlt_nview<4>(uu, pp, x);
  X[(int64_t)idx * 3 + 0] = x[0];
  X[(int64_t)idx * 3 + 1] = x[1];
  X[(int64_t)idx * 3 + 2] = x[2];
  if (status) status[idx] = st;
}

// img_utils.py:72-105 with its float32 roundings.  Returns the 2x3 transform
// mapping src->dst (inv=0: image->patch) or dst->src (inv=1: patch->image).
__host__ __device__ void patch_affine(const double* box, double patch_w, double patch_h, int inv,
                             double (&M)[2][3]) {
  const double c_x = box[0], c_y = box[1], scale = box[4], rot = box[5];
  const double src_w = box[2] * scale, src_h = box[3] * scale;
  const double rot_rad = 3.141592653589793 * rot / 180;
  const double sn = sin(rot_rad), cs = cos(rot_rad);
  // rotate_2d(np.array([0, src_h*0.5], f32), rot_rad) -> f32 (:63-69)
  const double dy_ = (double)(float)(src_h * 0.5), rx_ = (double)(float)(src_w * 0.5);
  const float down_x = (float)(0.0 * cs - dy_ * sn), down_y = (float)(0.0 * sn + dy_ * cs);
  const float right_x = (float)(rx_ * cs - 0.0 * sn), right_y = (float)(rx_ * sn + 0.0 * cs);
  float s[3][2], d[3][2];
  s[0][0] = (float)c_x;                       s[0][1] = (float)c_y;
  s[1][0] = (float)(c_x + (double)down_x);    s[1][1] = (float)(c_y + (double)down_y);
  s[2][0] = (float)(c_x + (double)right_x);   s[2][1] = (float)(c_y + (double)right_y);
  const float dcx = (float)(patch_w * 0.5), dcy = (float)(patch_h * 0.5);
  d[0][0] = dcx;        d[0][1] = dcy;
  d[1][0] = dcx + 0.f;  d[1][1] = dcy + (float)(patch_h * 0.5);
  d[2][0] = dcx + (float)(patch_w * 0.5);  d[2][1] = dcy + 0.f;
  const float (*from)[2] = inv ? d : s;
  const float (*to)[2] = inv ? s : d;
  // cv2.getAffineTransform: solve [x y 1] m = to, float64
  const double e1x = (double)from[1][0] - from[0][0], e1y = (double)from[1][1] - from[0][1];
  const double e2x = (double)from[2][0] - from[0][0], e2y = (double)from[2][1] - from[0][1];
  const double det = e1x * e2y - e1y * e2x;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const double f1 = (double)to[1][r] - to[0][r], f2 = (double)to[2][r] - to[0][r];
    const double a = (f1 * e2y - f2 * e1y) / det;
    const double b = (e1x * f2 - e2x * f1) / det;
    M[r][0] = a;
    M[r][1] = b;
    M[r][2] = (double)to[0][r] - a * from[0][0] - b * from[0][1];
  }
}

// One soft-argmax coordinate c [3] (normalised) of a sample with box [6] -> image point k [4] =
// (x px, y px, z mm, 1).  Shared by patch_to_image_kernel and the tuple-label entry.
__host__ __device__ inline void patch_to_image_point(const float* c, const double* box, double patch_w,
                                                     double patch_h, double rect3d_w, double* k) {
  // integral_loss.py:196-201
  const double px = ((double)c[0] + 0.5) * patch_w;
  const double py = ((double)c[1] + 0.5) * patch_h;
  const double pz = (double)c[2] * patch_w;
  double M[2][3];
  patch_affine(box, patch_w, patch_h, 1, M);
  // img_utils.py:108-111 np.dot(trans, [x, y, 1])
  k[0] = (M[0][0] * px + M[0][1] * py) + M[0][2];
  k[1] = (M[1][0] * px + M[1][1] * py) + M[1][2];
  k[2] = pz / patch_w * rect3d_w;  // img_utils.py:154
  k[3] = 1.0;
}

__global__ void patch_to_image_kernel(const float* __restrict__ coords,
                                      const double* __restrict__ box, int B, int J,
                                      double patch_w, double patch_h, double rect3d_w,
                                      double* __restrict__ kps) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * J) return;
  const int b = idx / J;
  patch_to_image_point(coords + idx * 3, box + b * 6, patch_w, patch_h, rect3d_w, kps + (int64_t)idx * 4);
}

// The label of one joint x [3] (world) in one view: root x0 [3] (joint 0, prep_h36m.py:181), c [16]
// = R(9) T(3) f(2) c(2), box [6].  Writes the label [3] and returns the camera-frame depths of the
// joint (cz) and of the root (pelvis_z).  Shared by project_labels_kernel and the tuple-label entry.
__host__ __device__ inline void project_label_point(const double* x, const double* x0, const double* c,
                                                    const double* box, double patch_w, double patch_h,
                                                    double rect3d_w, float* label, double& cz_out,
                                                    double& pelvis_z_out) {
  // prep_h36m.py:186 np.dot(rot, keypoints - trans)
  const double dx = x[0] - c[9], dy = x[1] - c[10], dz = x[2] - c[11];
  const double cx = (c[0] * dx + c[1] * dy) + c[2] * dz;
  const double cy = (c[3] * dx + c[4] * dy) + c[5] * dz;
  const double cz = (c[6] * dx + c[7] * dy) + c[8] * dz;
  const double rx = x0[0] - c[9], ry = x0[1] - c[10], rz = x0[2] - c[11];
  const double pelvis_z = (c[6] * rx + c[7] * ry) + c[8] * rz;
  // CamProj :170-175
  double u = cx / cz * c[12] + c[14];
  double v = cy / cz * c[13] + c[15];
  double z = cz - pelvis_z;  // :199
  double M[2][3];
  patch_affine(box, patch_w, patch_h, 0, M);
  const double pu = (M[0][0] * u + M[0][1] * v) + M[0][2];   // img_utils.py:235
  const double pv = (M[1][0] * u + M[1][1] * v) + M[1][2];
  z = z / (rect3d_w * box[4]) * patch_w;                       // :236
  // integral_loss.py:171-173
  label[0] = (float)(pu / patch_w - 0.5);
  label[1] = (float)(pv / patch_h - 0.5);
  label[2] = (float)(z / patch_w);
  cz_out = cz;
  pelvis_z_out = pelvis_z;
}

__global__ void project_labels_kernel(const double* __restrict__ X, const double* __restrict__ cam,
                                      const double* __restrict__ box, int B, int J,
                                      double patch_w, double patch_h, double rect3d_w,
                                      float* __restrict__ label, float* __restrict__ weight) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * J) return;
  const int b = idx / J;
  double cz, pz;
  project_label_point(X + (int64_t)idx * 3, X + (int64_t)b * J * 3, cam + b * 16, box + b * 6, patch_w,
                      patch_h, rect3d_w, label + idx * 3, cz, pz);
  weight[idx * 3 + 0] = 1.f;
  weight[idx * 3 + 1] = 1.f;
  weight[idx * 3 + 2] = 1.f;
}

// --------------------------------------------------------------- evaluation (H36M protocol)
// compute_similarity_transform(X, Y, compute_optimal_scale=True) (lib/utils/prep_h36m.py:108-168,
// numpy SVD there; here the one-sided Jacobi on the 3x3 covariance -- V*U^T does not depend on the
// ordering / paired signs of the singular triplets): X (targets) ~ b * Y (inputs) * T + c.
// X(j, o) / Y(j, o) write joint j of each pose into o[3]; they are called again for every pass
// over the joints, so a back-projecting caller never stores the camera-frame poses.
template <class GetX, class GetY>
__host__ __device__ inline void similarity_transform(int J, GetX X, GetY Y, double (&T)[3][3], double& bsc,
                                                     double (&cvec)[3]) {
  double muX[3] = {0, 0, 0}, muY[3] = {0, 0, 0};
  for (int j = 0; j < J; ++j) {
    double x[3], y[3];
    X(j, x);
    Y(j, y);
    for (int k = 0; k < 3; ++k) { muX[k] += x[k]; muY[k] += y[k]; }
  }
  for (int k = 0; k < 3; ++k) { muX[k] /= J; muY[k] /= J; }
  double ssX = 0, ssY = 0;
  for (int j = 0; j < J; ++j) {
    double x[3], y[3];
    X(j, x);
    Y(j, y);
    for (int k = 0; k < 3; ++k) {
      const double a = x[k] - muX[k], b = y[k] - muY[k];
      ssX += a * a;
      ssY += b * b;
    }
  }
  const double normX = sqrt(ssX), normY = sqrt(ssY);
  double A[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};     // X0^T Y0 (unit Frobenius norm each)
  for (int j = 0; j < J; ++j) {
    double x[3], y[3];
    X(j, x);
    Y(j, y);
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b)
        A[a][b] += ((x[a] - muX[a]) / normX) * ((y[b] - muY[b]) / normY);
  }
  double V[3][3];
  jacobi_onesided<3, 3>(A, V);                            // A = U diag(sg) (columns)
  double sg[3], U[3][3];
  for (int c = 0; c < 3; ++c) {
    sg[c] = sqrt(A[0][c] * A[0][c] + A[1][c] * A[1][c] + A[2][c] * A[2][c]);
    for (int r = 0; r < 3; ++r) U[r][c] = sg[c] > 0 ? A[r][c] / sg[c] : 0.0;
  }
  int jmin = 0;
  for (int c = 1; c < 3; ++c) if (sg[c] < sg[jmin]) jmin = c;
  if (sg[jmin] == 0.0) {
    // rank-deficient covariance: complete U with the cross product of the other two columns
    const int a = (jmin + 1) % 3, b = (jmin + 2) % 3;
    U[0][jmin] = U[1][a] * U[2][b] - U[2][a] * U[1][b];
    U[1][jmin] = U[2][a] * U[0][b] - U[0][a] * U[2][b];
    U[2][jmin] = U[0][a] * U[1][b] - U[1][a] * U[0][b];
  }
  auto make_T = [&]() {
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c)
        T[r][c] = V[r][0] * U[c][0] + V[r][1] * U[c][1] + V[r][2] * U[c][2];   // V U^T
  };
  make_T();
  const double det = T[0][0] * (T[1][1] * T[2][2] - T[1][2] * T[2][1]) -
                     T[0][1] * (T[1][0] * T[2][2] - T[1][2] * T[2][0]) +
                     T[0][2] * (T[1][0] * T[2][1] - T[1][1] * T[2][0]);
  const double sgn = det > 0 ? 1.0 : (det < 0 ? -1.0 : 0.0);   // np.sign
  for (int r = 0; r < 3; ++r) V[r][jmin] *= sgn;               // V[:,-1] *= sign(detT)
  sg[jmin] *= sgn;
  make_T();
  const double trace = sg[0] + sg[1] + sg[2];
  bsc = trace * normX / normY;                                 // optimal scale
  for (int c = 0; c < 3; ++c)
    cvec[c] = muX[c] - bsc * (muY[0] * T[0][c] + muY[1] * T[1][c] + muY[2] * T[2][c]);
}

// lib/dataset/h36m.py:168-378 per sample: back-projection of image-space joints
// (lib/utils/prep_h36m.py:85-89), similarity alignment with optimal scale, root alignment and
// the nine protocol means.  One thread per sample, float64, J <= 32.
//   metrics[s] = { e, e_align, e_norm, e14, e14_align, e14_norm, ex, ey, ez }   (means over joints)
// (also compiled for the host: tests/harness/host_geometry.cu runs this exact code on the CPU)
__host__ __device__ void h36m_eval_sample(const double* p, const double* q, const double* cam,
                                          int J, int root, unsigned j14mask, double pck_thr,
                                          double* metrics, double* per_joint, int32_t* pck,
                                          double* poses) {
  // back projection (h36m.py:228-240): X = gt (targets), Y = prediction (inputs)
  auto bp = [&](const double* a, int j, double (&o)[3]) { cam_back_proj(a, j, cam, o); };
  double T[3][3], bsc, cvec[3];
  similarity_transform(J, [&](int j, double (&o)[3]) { bp(q, j, o); },
                       [&](int j, double (&o)[3]) { bp(p, j, o); }, T, bsc, cvec);
  // root joint of each variant (h36m.py:247-251)
  double xr[3], yr[3], yar[3], ynr[3];
  bp(q, root, xr);
  bp(p, root, yr);
  for (int c = 0; c < 3; ++c) {
    yar[c] = bsc * (yr[0] * T[0][c] + yr[1] * T[1][c] + yr[2] * T[2][c]) + cvec[c];
    ynr[c] = bsc * yr[c];
  }
  double m[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  int n14 = 0;
  for (int j = 0; j < J; ++j) {
    double x[3], y[3], d[3], da[3], dn[3];
    bp(q, j, x);
    bp(p, j, y);
    for (int c = 0; c < 3; ++c) {
      const double ya = bsc * (y[0] * T[0][c] + y[1] * T[1][c] + y[2] * T[2][c]) + cvec[c];
      const double yn = bsc * y[c];
      const double g0 = x[c] - xr[c];
      d[c] = g0 - (y[c] - yr[c]);
      da[c] = g0 - (ya - yar[c]);
      dn[c] = g0 - (yn - ynr[c]);
      if (poses) {
        double* o = poses + j * 9;
        o[c] = y[c] - yr[c];            // pred
        o[3 + c] = ya - yar[c];         // align_pred
        o[6 + c] = g0;                  // gt
      }
    }
    const double e = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    const double ea = sqrt(da[0] * da[0] + da[1] * da[1] + da[2] * da[2]);
    const double en = sqrt(dn[0] * dn[0] + dn[1] * dn[1] + dn[2] * dn[2]);
    m[0] += e; m[1] += ea; m[2] += en;
    if ((j14mask >> j) & 1u) { m[3] += e; m[4] += ea; m[5] += en; ++n14; }
    m[6] += fabs(d[0]); m[7] += fabs(d[1]); m[8] += fabs(d[2]);
    if (per_joint) per_joint[j] = e;
    if (pck) pck[j] = e >= pck_thr ? 0 : 1;
  }
  for (int k = 0; k < 9; ++k) {
    const int div = (k >= 3 && k < 6) ? (n14 > 0 ? n14 : 1) : J;
    metrics[k] = m[k] / div;
  }
}

__global__ void h36m_eval_kernel(const double* __restrict__ pred, const double* __restrict__ gt,
                                 const double* __restrict__ cam, int S, int J, int root,
                                 unsigned j14mask, double pck_thr, double* __restrict__ metrics,
                                 double* __restrict__ per_joint, int32_t* __restrict__ pck,
                                 double* __restrict__ poses) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  h36m_eval_sample(pred + (int64_t)s * J * 3, gt + (int64_t)s * J * 3, cam + (int64_t)s * 5, J, root,
                   j14mask, pck_thr, metrics + (int64_t)s * 9,
                   per_joint ? per_joint + (int64_t)s * J : nullptr,
                   pck ? pck + (int64_t)s * J : nullptr,
                   poses ? poses + (int64_t)s * J * 9 : nullptr);
}

// Per-sample errors of camera-frame poses (the refiner's evaluate, refiner/data.py:78-160 of the
// reference): no back-projection and no root alignment; X = gt, Y = pred.  float64, J <= 32.
//   metrics[7] = { e, e_align, e_sub, e_align_sub, |dx|, |dy|, |dz| }   (means over joints)
// (also compiled for the host: tests/harness/host_pose_eval.cu)
__host__ __device__ void pose_errors_sample(const double* p, const double* q, int J, unsigned submask,
                                            double* metrics, double* per_joint) {
  double T[3][3], bsc, cvec[3];
  auto at = [](const double* a) {
    return [a](int j, double (&o)[3]) { o[0] = a[j * 3]; o[1] = a[j * 3 + 1]; o[2] = a[j * 3 + 2]; };
  };
  similarity_transform(J, at(q), at(p), T, bsc, cvec);
  double m[7] = {0, 0, 0, 0, 0, 0, 0};
  int nsub = 0;
  for (int j = 0; j < J; ++j) {
    const double* x = q + j * 3;
    const double* y = p + j * 3;
    double d[3], da[3];
    for (int c = 0; c < 3; ++c) {
      const double ya = bsc * (y[0] * T[0][c] + y[1] * T[1][c] + y[2] * T[2][c]) + cvec[c];
      d[c] = x[c] - y[c];
      da[c] = x[c] - ya;
    }
    const double e = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    const double ea = sqrt(da[0] * da[0] + da[1] * da[1] + da[2] * da[2]);
    m[0] += e; m[1] += ea;
    if ((submask >> j) & 1u) { m[2] += e; m[3] += ea; ++nsub; }
    m[4] += fabs(d[0]); m[5] += fabs(d[1]); m[6] += fabs(d[2]);
    if (per_joint) per_joint[j] = e;
  }
  for (int k = 0; k < 7; ++k) {
    const int div = (k == 2 || k == 3) ? (nsub > 0 ? nsub : 1) : J;
    metrics[k] = m[k] / div;
  }
}

__global__ void pose_errors_kernel(const double* __restrict__ pred, const double* __restrict__ gt, int S, int J,
                                   unsigned submask, double* __restrict__ metrics,
                                   double* __restrict__ per_joint) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  pose_errors_sample(pred + (int64_t)s * J * 3, gt + (int64_t)s * J * 3, J, submask, metrics + (int64_t)s * 7,
                     per_joint ? per_joint + (int64_t)s * J : nullptr);
}

// Root-relative camera-frame pose of image-space joints: the `pred` column of h36m_eval_sample's
// poses, with the same arithmetic (CamBackProj of joint j minus CamBackProj of the root).
__host__ __device__ void pose_to_camera_sample(const double* a, const double* cam, int J, int root, double* out) {
  double r[3];
  cam_back_proj(a, root, cam, r);
  for (int j = 0; j < J; ++j) {
    double y[3];
    cam_back_proj(a, j, cam, y);
    for (int c = 0; c < 3; ++c) out[j * 3 + c] = y[c] - r[c];
  }
}

__global__ void pose_to_camera_kernel(const double* __restrict__ joints, const double* __restrict__ cam, int N,
                                      int J, int root, double* __restrict__ out) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= N) return;
  pose_to_camera_sample(joints + (int64_t)s * J * 3, cam + (int64_t)s * 5, J, root, out + (int64_t)s * J * 3);
}

// --------------------------------------------------------------- pseudo-label records
// One thread per (frame, camera), cam_pseudo_record (camera.cuh) over its J joints.  X holds S
// poses per frame: S = 1 serves every camera, S = V one pose per camera.  Every offset is derived
// from the sizes the entry validated; nothing read from X or status indexes memory.
__global__ void pseudo_records_kernel(const double* __restrict__ X, const int32_t* __restrict__ status,
                                      const double* __restrict__ cam, int T, int S, int V, int J, int root,
                                      double* __restrict__ jt, double* __restrict__ vis,
                                      double* __restrict__ pelvis, int32_t* __restrict__ ok) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)T * V) return;
  const int64_t t = i / V, v = i % V;
  const int64_t s = t * S + (S == 1 ? 0 : v);
  ok[i] = cam_pseudo_record(X + s * J * 3, status + s * J, cam + i * 16, J, root, jt + i * J * 3, vis + i * J * 3,
                            pelvis + i * 3);
}

// The size checks of epb_pseudo_records, on the host before any launch.
int pseudo_records_sizes(int T, int S, int V, int J, int root) {
  EPB_CHECK_ARG(T >= 0 && S >= 0 && V >= 0 && J >= 0);
  EPB_CHECK_ARG(V >= 2 && V <= 8 && (S == 1 || S == V));
  EPB_CHECK_ARG(root >= 0 && root < J);
  EPB_CHECK_ARG((int64_t)T * V * J <= 0x7fffffff);
  return EPB_OK;
}

// --------------------------------------------------------------- relative pose (no extrinsics)
// Self-supervision without camera extrinsics: the geometry of a view pair comes from its own
// predicted 2-D joints.  The reference leaves only the pieces (lib/utils/cameras.py:133-143,
// Camera.get_essential_matrix / get_fundamental_matrix with cv2.FM_LMEDS, no caller); per pair
// (a = sample i, b = sample i + B/2):
//   1. robust F by least median of squares: RP_HYP hypotheses, each fundamental_8point on 8
//      distinct joints, scored by the lower median over all J joints of the squared Sampson
//      distance (px^2); best = lowest score, ties to the lowest hypothesis; inliers r^2 <=
//      max((2.5 sigma)^2, (1e-3 px)^2), sigma = 1.4826 (1 + 5/(J-8)) sqrt(score); refit
//      fundamental_8point on the inliers.  DEPARTURES from cv2.findFundamentalMat(FM_LMEDS):
//      the joints of hypothesis h are a FIXED schedule (the first 8 entries of a Fisher-Yates
//      shuffle of 0..J-1 driven by splitmix64 seeded with h), the same for every pair and step,
//      so the estimate is deterministic (cv2 draws them at random); the points are not
//      truncated to integers as the reference's np.int32 cast does.  256 hypotheses draw an
//      outlier-free 8-set with 99.9 % probability at 6 outliers among 17 joints.
//   2. E = K_b^T F K_a; E = U diag(s) V^T by the one-sided Jacobi SVD, columns ordered by
//      decreasing s, u3 = u1 x u2 and v3 = v1 x v2 (det U = det V = +1) and the sign of the
//      pair (u1, v1) chosen so that the largest-magnitude entry of u3 is positive (this makes
//      the candidate order independent of the SVD's sign conventions).  Candidates, in order:
//      (U W V^T, u3), (U W V^T, -u3), (U W^T V^T, u3), (U W^T V^T, -u3); the one with the most
//      DLT-triangulated inliers in front of both cameras wins (ties to the first).
//   3. scale (our rule; the reference has none): with |t| = 1 the root joint (0) is
//      triangulated at depths Z_a, Z_b; s_v = f_x,v rect3d_w / (bb_w,v scale_v Z_v) is the scale
//      at which the box spans rect3d_w mm at the root's depth -- the assumption the label
//      arithmetic of project_labels_kernel already makes -- and t <- sqrt(s_a s_b) t.
//   4. P_a = K_a [I|0], P_b = K_b [R|t]; cam rows a: R = I, T = 0; b: R, T = -R^T t.
// status 0 (R = I, t = 0, no NaN in any output) for: no valid hypothesis, fewer than 8
// inliers, a failed refit, fewer than max(8, ceil(n_inl/2)) inliers in front for the winner,
// Z_a <= 0 or Z_b <= 0, or any non-finite value.  The body is shared by the kernel (one warp per
// pair: lanes split the hypotheses and the cheirality DLTs) and the CPU harness (one lane).
constexpr int RP_HYP = 256;
constexpr int RP_MAXJ = 32;

__host__ __device__ inline uint64_t splitmix64_next(uint64_t& s) {
  uint64_t z = (s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__host__ __device__ inline bool finite2(const double* p) {
  return isfinite(p[0]) && isfinite(p[1]);
}

// hypothesis h: fundamental_8point on its 8 scheduled joints (false: a non-finite joint or no F)
__host__ __device__ inline bool relpose_hypothesis(const double* ua, const double* ub, int su, int J,
                                                   int h, double* F) {
  int perm[RP_MAXJ];
  for (int i = 0; i < J; ++i) perm[i] = i;
  uint64_t s = (uint64_t)h;
  double a[16], b[16];
  for (int k = 0; k < 8; ++k) {
    const int r = k + (int)(splitmix64_next(s) % (uint64_t)(J - k));
    const int t = perm[k];
    perm[k] = perm[r];
    perm[r] = t;
    const double* pa = ua + (int64_t)perm[k] * su;
    const double* pb = ub + (int64_t)perm[k] * su;
    if (!finite2(pa) || !finite2(pb)) return false;
    a[2 * k] = pa[0]; a[2 * k + 1] = pa[1];
    b[2 * k] = pb[0]; b[2 * k + 1] = pb[1];
  }
  return fundamental_8point(a, b, 2, 8, F);
}

// squared Sampson distance (px^2) of the match (a, b) to F; +inf when not finite
__host__ __device__ inline double sampson2(const double* F, const double* a, const double* b) {
  const double x1 = a[0], y1 = a[1], x2 = b[0], y2 = b[1];
  const double f0 = (F[0] * x1 + F[1] * y1) + F[2];       // F (x1, y1, 1)
  const double f1 = (F[3] * x1 + F[4] * y1) + F[5];
  const double f2 = (F[6] * x1 + F[7] * y1) + F[8];
  const double g0 = (F[0] * x2 + F[3] * y2) + F[6];       // F^T (x2, y2, 1)
  const double g1 = (F[1] * x2 + F[4] * y2) + F[7];
  const double e = (x2 * f0 + y2 * f1) + f2;
  const double r = e * e / (((f0 * f0 + f1 * f1) + g0 * g0) + g1 * g1);
  return isfinite(r) ? r : INFINITY;
}

// lower median over the J joints of the squared Sampson distance
__host__ __device__ inline double relpose_score(const double* F, const double* ua, const double* ub,
                                                int su, int J) {
  double r[RP_MAXJ];
  for (int j = 0; j < J; ++j) {
    const double v = sampson2(F, ua + (int64_t)j * su, ub + (int64_t)j * su);
    int i = j;
    for (; i > 0 && r[i - 1] > v; --i) r[i] = r[i - 1];
    r[i] = v;
  }
  return r[(J - 1) / 2];
}

// per-lane reductions of relpose_pair: one lane on the host, a full warp on the device
struct RpSerial {
  int lane = 0, n = 1;
  __host__ __device__ void argmin(double&, int&) const {}
  __host__ __device__ int sum(int v) const { return v; }
};
struct RpWarp {
  int lane, n = 32;
  __host__ __device__ void argmin(double& s, int& h) const {
#ifdef __CUDA_ARCH__
    for (int o = 16; o > 0; o >>= 1) {
      const double os = __shfl_xor_sync(0xffffffffu, s, o);
      const int oh = __shfl_xor_sync(0xffffffffu, h, o);
      if (os < s || (os == s && oh < h)) { s = os; h = oh; }
    }
#endif
  }
  __host__ __device__ int sum(int v) const {
#ifdef __CUDA_ARCH__
    return __reduce_add_sync(0xffffffffu, v);
#else
    return v;
#endif
  }
};

// candidate c of the decomposition: R (row-major) and unit t
__host__ __device__ inline void relpose_candidate(const double (&R1)[9], const double (&R2)[9],
                                                  const double (&u3)[3], int c, double* R, double* t) {
  for (int k = 0; k < 9; ++k) R[k] = c < 2 ? R1[k] : R2[k];
  const double sg = (c & 1) ? -1.0 : 1.0;
  for (int k = 0; k < 3; ++k) t[k] = sg * u3[k];
}

// K [R|t] (row-major 3x4) from intrinsics f(2) c(2)
__host__ __device__ inline void relpose_P(const double* in, const double* R, const double* t, double* P) {
  for (int k = 0; k < 4; ++k) {
    const double r0 = k < 3 ? R[k] : t[0], r1 = k < 3 ? R[3 + k] : t[1], r2 = k < 3 ? R[6 + k] : t[2];
    P[k] = in[0] * r0 + in[2] * r2;
    P[4 + k] = in[1] * r1 + in[3] * r2;
    P[8 + k] = r2;
  }
}

// DLT of joint j with P_a = K_a[I|0], P_b = K_b[R|t]; returns the two depths
__host__ __device__ inline bool relpose_depths(const double* ua, const double* ub, const double* Pab,
                                               const double* R, const double* t, double& za,
                                               double& zb) {
  const double uu[4] = {ua[0], ua[1], ub[0], ub[1]};
  double x[3];
  const int st = dlt_nview<2>(uu, Pab, x);
  za = x[2];
  zb = ((R[6] * x[0] + R[7] * x[1]) + R[8] * x[2]) + t[2];
  return st != 0;
}

// One view pair.  ia / ib: f(2) c(2); box: c_x c_y w h scale rot.  Outputs as epb_relative_pose;
// diag (may be null): chosen hypothesis (-1: none), chosen candidate (-1: none), inlier count.
template <class Red>
__host__ __device__ void relpose_pair(const Red& red, const double* ua, const double* ub, int su, int J,
                                      const double* ia, const double* ib, const double* boxa,
                                      const double* boxb, double rect3d_w, double* Pa, double* Pb,
                                      double* cama, double* camb, int32_t* inl, int32_t* status,
                                      int32_t* diag) {
  // 1. hypotheses: lane l scores h = l, l + n, ...; (score, h) minimum across the lanes
  double best = INFINITY;
  int bh = RP_HYP;
  for (int h = red.lane; h < RP_HYP; h += red.n) {
    double F[9];
    if (!relpose_hypothesis(ua, ub, su, J, h, F)) continue;
    const double s = relpose_score(F, ua, ub, su, J);
    if (s < best) { best = s; bh = h; }
  }
  red.argmin(best, bh);
  // every lane repeats the (cheap, identical) serial part, so `ok` is warp-uniform
  bool ok = bh < RP_HYP;
  double F[9];
  unsigned mask = 0u;
  int n_inl = 0;
  if (ok) {
    relpose_hypothesis(ua, ub, su, J, bh, F);
    const double sig = J > 8 ? 1.4826 * (1.0 + 5.0 / (J - 8)) * sqrt(best) : INFINITY;
    const double thr = J > 8 ? fmax(2.5 * sig * (2.5 * sig), 1e-6) : DBL_MAX;
    for (int j = 0; j < J; ++j)
      if (sampson2(F, ua + (int64_t)j * su, ub + (int64_t)j * su) <= thr) { mask |= 1u << j; ++n_inl; }
  }
  ok = ok && n_inl >= 8;
  if (ok) {                                            // refit on the inliers
    double ga[2 * RP_MAXJ], gb[2 * RP_MAXJ];
    int n = 0;
    for (int j = 0; j < J; ++j)
      if ((mask >> j) & 1u) {
        ga[2 * n] = ua[(int64_t)j * su]; ga[2 * n + 1] = ua[(int64_t)j * su + 1];
        gb[2 * n] = ub[(int64_t)j * su]; gb[2 * n + 1] = ub[(int64_t)j * su + 1];
        ++n;
      }
    ok = fundamental_8point(ga, gb, 2, n, F);
  }
  // 2. E = K_b^T F K_a and its decomposition
  double R1[9], R2[9], u3[3];
  if (ok) {
    const double Ka[3][3] = {{ia[0], 0, ia[2]}, {0, ia[1], ia[3]}, {0, 0, 1}};
    const double Kb[3][3] = {{ib[0], 0, ib[2]}, {0, ib[1], ib[3]}, {0, 0, 1}};
    double M[3][3], A[3][3], V[3][3];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j)
        M[i][j] = (F[i * 3 + 0] * Ka[0][j] + F[i * 3 + 1] * Ka[1][j]) + F[i * 3 + 2] * Ka[2][j];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        A[i][j] = (Kb[0][i] * M[0][j] + Kb[1][i] * M[1][j]) + Kb[2][i] * M[2][j];
        ok = ok && isfinite(A[i][j]);
      }
    if (ok) {
      jacobi_onesided<3, 3>(A, V);
      double sg[3];
      for (int c = 0; c < 3; ++c) sg[c] = sqrt(A[0][c] * A[0][c] + A[1][c] * A[1][c] + A[2][c] * A[2][c]);
      int o0 = 0, o1 = 1, o2 = 2, tmp;                   // stable sort, decreasing
      if (sg[o1] > sg[o0]) { tmp = o0; o0 = o1; o1 = tmp; }
      if (sg[o2] > sg[o1]) { tmp = o1; o1 = o2; o2 = tmp; }
      if (sg[o1] > sg[o0]) { tmp = o0; o0 = o1; o1 = tmp; }
      double u1[3], u2[3], v1[3], v2[3], v3[3];
      for (int r = 0; r < 3; ++r) {
        u1[r] = A[r][o0] / sg[o0]; u2[r] = A[r][o1] / sg[o1];
        v1[r] = V[r][o0]; v2[r] = V[r][o1];
      }
      u3[0] = u1[1] * u2[2] - u1[2] * u2[1];
      u3[1] = u1[2] * u2[0] - u1[0] * u2[2];
      u3[2] = u1[0] * u2[1] - u1[1] * u2[0];
      v3[0] = v1[1] * v2[2] - v1[2] * v2[1];
      v3[1] = v1[2] * v2[0] - v1[0] * v2[2];
      v3[2] = v1[0] * v2[1] - v1[1] * v2[0];
      int km = 0;
      for (int k = 1; k < 3; ++k) if (fabs(u3[k]) > fabs(u3[km])) km = k;
      if (u3[km] < 0) {
        for (int k = 0; k < 3; ++k) { u1[k] = -u1[k]; v1[k] = -v1[k]; u3[k] = -u3[k]; v3[k] = -v3[k]; }
      }
      // U W V^T = u2 v1^T - u1 v2^T + u3 v3^T,  U W^T V^T = -u2 v1^T + u1 v2^T + u3 v3^T
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
          const double p = u2[i] * v1[j] - u1[i] * v2[j], q = u3[i] * v3[j];
          R1[i * 3 + j] = p + q;
          R2[i * 3 + j] = q - p;
          ok = ok && isfinite(R1[i * 3 + j]) && isfinite(R2[i * 3 + j]);
        }
    }
  }
  // cheirality: lanes split the (candidate, joint) DLTs
  const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, z3[3] = {0, 0, 0};
  double Pab[24];
  relpose_P(ia, I3, z3, Pab);
  int cnt[4] = {0, 0, 0, 0};
  const bool cheir = ok;
  if (ok) {
    for (int i = red.lane; i < 4 * J; i += red.n) {
      const int c = i / J, j = i - c * J;
      if (!((mask >> j) & 1u)) continue;
      double R[9], t[3], za, zb;
      relpose_candidate(R1, R2, u3, c, R, t);
      relpose_P(ib, R, t, Pab + 12);
      if (relpose_depths(ua + (int64_t)j * su, ub + (int64_t)j * su, Pab, R, t, za, zb) && za > 0 && zb > 0)
        ++cnt[c];
    }
  }
  int win = 0;
  for (int c = 0; c < 4; ++c) {
    cnt[c] = red.sum(cnt[c]);
    if (cnt[c] > cnt[win]) win = c;
  }
  ok = ok && cnt[win] >= (n_inl + 1) / 2 && cnt[win] >= 8;
  // 3. scale from the root joint
  double R[9], t[3];
  relpose_candidate(R1, R2, u3, win, R, t);
  if (ok) {
    double za, zb;
    relpose_P(ib, R, t, Pab + 12);
    ok = relpose_depths(ua, ub, Pab, R, t, za, zb) && za > 0 && zb > 0;
    if (ok) {
      const double sa = ia[0] * rect3d_w / (boxa[2] * boxa[4] * za);
      const double sb = ib[0] * rect3d_w / (boxb[2] * boxb[4] * zb);
      const double s = sqrt(sa * sb);
      for (int k = 0; k < 3; ++k) t[k] *= s;
    }
  }
  // 4. outputs
  double pb[12], T[3];
  if (ok) {
    relpose_P(ib, R, t, pb);
    for (int k = 0; k < 3; ++k) T[k] = -((R[k] * t[0] + R[3 + k] * t[1]) + R[6 + k] * t[2]);
    for (int k = 0; k < 12; ++k) ok = ok && isfinite(pb[k]) && isfinite(Pab[k]);
    for (int k = 0; k < 3; ++k) ok = ok && isfinite(T[k]);
  }
  if (!ok) {
    for (int k = 0; k < 9; ++k) R[k] = I3[k];
    for (int k = 0; k < 3; ++k) { t[k] = 0.0; T[k] = 0.0; }
    relpose_P(ib, R, t, pb);
  }
  if (red.lane != 0) return;
  for (int k = 0; k < 12; ++k) { Pa[k] = Pab[k]; Pb[k] = pb[k]; }
  for (int k = 0; k < 9; ++k) { cama[k] = I3[k]; camb[k] = R[k]; }
  for (int k = 0; k < 3; ++k) { cama[9 + k] = 0.0; camb[9 + k] = T[k]; }
  for (int k = 0; k < 4; ++k) { cama[12 + k] = ia[k]; camb[12 + k] = ib[k]; }
  for (int j = 0; j < J; ++j) inl[j] = (mask >> j) & 1u;
  *status = ok ? 1 : 0;
  if (diag) {
    diag[0] = bh < RP_HYP ? bh : -1;
    diag[1] = cheir ? win : -1;
    diag[2] = n_inl;
  }
}

// u [B][J][stride_u], intr [B][4], box [B][6]; one warp per pair i = (i, i + NP)
__global__ void relative_pose_kernel(const double* __restrict__ u, int stride_u,
                                     const double* __restrict__ intr, const double* __restrict__ box,
                                     int NP, int J, double rect3d_w, double* __restrict__ Pa,
                                     double* __restrict__ Pb, double* __restrict__ cam,
                                     int32_t* __restrict__ inl, int32_t* __restrict__ status,
                                     int32_t* __restrict__ diag) {
  const int pair = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (pair >= NP) return;                                  // warp-uniform
  RpWarp red;
  red.lane = threadIdx.x & 31;
  const int a = pair, b = pair + NP;
  relpose_pair(red, u + (int64_t)a * J * stride_u, u + (int64_t)b * J * stride_u, stride_u, J,
               intr + a * 4, intr + b * 4, box + a * 6, box + b * 6, rect3d_w, Pa + pair * 12,
               Pb + pair * 12, cam + a * 16, cam + b * 16, inl + (int64_t)pair * J, status + pair,
               diag ? diag + pair * 3 : nullptr);
}

// --------------------------------------------------------------- robust V-view triangulation
// Inference on a calibrated rig (2 <= V <= 8 views; not in the reference, which only pairs two
// views): per (tuple, joint) a consensus over the view pairs instead of one DLT over all views, so
// that a wrong 2-D joint in one view (occlusion, left / right swap) is left out and reported.
//   usable views: weight > 0 (and finite) and a finite image point.
//   1. hypotheses: every pair of usable views in the order (0,1), (0,2), .., (V-2,V-1) (<= 28),
//      each dlt_nview<2>.
//   2. score: a usable view is an inlier when the hypothesis lies in front of it (third row of P
//      times (X, 1) > 0) and reprojects within thr px; cost = sum over the usable views of e^2 for
//      inliers and thr^2 otherwise (MSAC).  Best = most inliers, then lowest cost, then lowest
//      hypothesis index: a total order, so the choice does not depend on the reduction's shape.
//   3. refit: DLT over the inlier views, rows scaled by the weights; the inlier set is taken again
//      against the refit point and, when it changed, the fit repeated once on the new set.
//   4. inliers = the views of the last fit, resid = RMS reprojection error (px) over them.
// status 0 with X = 0, inliers = 0, resid = 0 for: fewer than two inlier views at any stage, a
// refit system of rank < 3 (the views' rays are one line), a non-finite coordinate or residual,
// |coordinate| > 1e16.  The body is shared by the kernel (one
// warp per (tuple, joint): lane h owns hypothesis h, every lane repeats the refit) and the CPU
// harness (one lane).
constexpr int RB_MAXV = 8;

struct RbSerial {
  int lane = 0, n = 1;
  __host__ __device__ void best(int&, double&, int&) const {}
};
struct RbWarp {
  int lane, n = 32;
  __host__ __device__ void best(int& cnt, double& cost, int& h) const {
#ifdef __CUDA_ARCH__
    for (int o = 16; o > 0; o >>= 1) {
      const int oc = __shfl_xor_sync(0xffffffffu, cnt, o);
      const double os = __shfl_xor_sync(0xffffffffu, cost, o);
      const int oh = __shfl_xor_sync(0xffffffffu, h, o);
      if (oc > cnt || (oc == cnt && (os < cost || (os == cost && oh < h)))) { cnt = oc; cost = os; h = oh; }
    }
#endif
  }
};

__host__ __device__ inline int robust_count(unsigned m) {
  int n = 0;
  for (; m; m &= m - 1) ++n;
  return n;
}

// views (a, b) of hypothesis h, generated from V
__host__ __device__ inline void robust_pair_of(int h, int V, int& a, int& b) {
  a = 0;
  while (h >= V - 1 - a) { h -= V - 1 - a; ++a; }
  b = a + 1 + h;
}

// squared reprojection error (px^2) of x in one view; false when x is not in front of the camera
// or the error is not finite
__host__ __device__ inline bool robust_reproj2(const double* u, const double* P, const double* x,
                                               double& e2) {
  const double z = ((P[8] * x[0] + P[9] * x[1]) + P[10] * x[2]) + P[11];
  const double dx = (((P[0] * x[0] + P[1] * x[1]) + P[2] * x[2]) + P[3]) / z - u[0];
  const double dy = (((P[4] * x[0] + P[5] * x[1]) + P[6] * x[2]) + P[7]) / z - u[1];
  e2 = dx * dx + dy * dy;
  return z > 0.0 && isfinite(e2);
}

// inlier views of x among `usable` and the MSAC cost over the usable views
__host__ __device__ inline unsigned robust_inliers(const double* u, const double* P, int V,
                                                   unsigned usable, const double* x, double thr2,
                                                   double& cost) {
  unsigned m = 0u;
  cost = 0.0;
  for (int v = 0; v < V; ++v) {
    if (!((usable >> v) & 1u)) continue;
    double e2;
    const bool in = robust_reproj2(u + 2 * v, P + 12 * v, x, e2) && e2 <= thr2;
    if (in) m |= 1u << v;
    cost += in ? e2 : thr2;
  }
  return m;
}

// the two-view DLT of hypothesis h (false: a view of the pair is not usable, or no finite point)
__host__ __device__ inline bool robust_hypothesis(const double* u, const double* P, int V,
                                                  unsigned usable, int h, double* x) {
  int a, b;
  robust_pair_of(h, V, a, b);
  if (!((usable >> a) & 1u) || !((usable >> b) & 1u)) return false;
  const double uu[4] = {u[2 * a], u[2 * a + 1], u[2 * b], u[2 * b + 1]};
  double pp[24];
  for (int k = 0; k < 12; ++k) { pp[k] = P[12 * a + k]; pp[12 + k] = P[12 * b + k]; }
  return dlt_nview<2>(uu, pp, x) != 0;
}

// weighted DLT over the views of `mask` (a view outside it contributes two rows of zeros, which
// change no sum of the Jacobi sweeps: with weights 1 and two views this is dlt_nview<2> bit for bit)
template <int VM>
__host__ __device__ inline bool dlt_masked(const double* u, const double* P, const double* w, int V,
                                           unsigned mask, double* x) {
  double A[2 * VM][4], Vm[4][4];
  for (int v = 0; v < VM; ++v) {
    const bool on = v < V && ((mask >> v) & 1u);
    for (int k = 0; k < 4; ++k) {
      A[2 * v + 0][k] = on ? w[v] * (u[v * 2 + 0] * P[v * 12 + 8 + k] - P[v * 12 + 0 + k]) : 0.0;
      A[2 * v + 1][k] = on ? w[v] * (u[v * 2 + 1] * P[v * 12 + 8 + k] - P[v * 12 + 4 + k]) : 0.0;
    }
  }
  jacobi_onesided<2 * VM, 4>(A, Vm);
  int best = 0;
  double bn = DBL_MAX, n2s[4], big = 0.0;
  for (int j = 0; j < 4; ++j) {
    double n2 = 0;
    for (int i = 0; i < 2 * VM; ++i) n2 += A[i][j] * A[i][j];
    n2s[j] = n2;
    big = fmax(big, n2);
    if (n2 < bn) { bn = n2; best = j; }
  }
  // rank 3 or the point is not determined (all rays the same line: identical cameras): the second
  // smallest singular value must stand clear of rounding, sigma > 1e-10 sigma_max
  double second = DBL_MAX;
  for (int j = 0; j < 4; ++j)
    if (j != best) second = fmin(second, n2s[j]);
  if (!(second > 1e-20 * big)) return false;
  double h[4];
  for (int i = 0; i < 4; ++i) {
    h[i] = Vm[i][0];
    for (int j = 1; j < 4; ++j)
      if (best == j) h[i] = Vm[i][j];
  }
  x[0] = h[0] / h[3]; x[1] = h[1] / h[3]; x[2] = h[2] / h[3];
  const double mx = fmax(fabs(x[0]), fmax(fabs(x[1]), fabs(x[2])));
  return isfinite(x[0]) && isfinite(x[1]) && isfinite(x[2]) && mx <= 1.e16;
}

// One (tuple, joint): u [V][2], P [V][12], w [V] (non-negative), 2 <= V <= RB_MAXV.
template <class Red>
__host__ __device__ void robust_point(const Red& red, const double* u, const double* P,
                                      const double* w, int V, double thr, double* X, int32_t* inl,
                                      double* resid, int32_t* status) {
  const double thr2 = thr * thr;
  unsigned usable = 0u;
  for (int v = 0; v < V; ++v)
    if (w[v] > 0.0 && isfinite(w[v]) && finite2(u + 2 * v)) usable |= 1u << v;
  // 1. + 2.: lane l scores hypotheses l, l + n, ..; the best (count, cost, h) across the lanes
  const int nh = V * (V - 1) / 2;
  int bn = -1, bh = nh;
  double bc = INFINITY;
  for (int h = red.lane; h < nh; h += red.n) {
    double x[3], c;
    if (!robust_hypothesis(u, P, V, usable, h, x)) continue;
    const int n = robust_count(robust_inliers(u, P, V, usable, x, thr2, c));
    if (n > bn || (n == bn && c < bc)) { bn = n; bc = c; bh = h; }
  }
  red.best(bn, bc, bh);
  // 3.: every lane repeats the (identical) refit, so `ok` is warp-uniform
  bool ok = bn >= 2;
  double x[3] = {0.0, 0.0, 0.0}, r = 0.0;
  unsigned mask = 0u;
  if (ok) {
    double c;
    robust_hypothesis(u, P, V, usable, bh, x);
    mask = robust_inliers(u, P, V, usable, x, thr2, c);
    auto refit = [&](unsigned m) {
      return V <= 4 ? dlt_masked<4>(u, P, w, V, m, x) : dlt_masked<RB_MAXV>(u, P, w, V, m, x);
    };
    ok = refit(mask);
    if (ok) {
      const unsigned m1 = robust_inliers(u, P, V, usable, x, thr2, c);
      if (m1 != mask) {
        mask = m1;
        ok = robust_count(m1) >= 2 && refit(m1);
      }
    }
    if (ok) {                                              // 4.
      double s2 = 0.0;
      for (int v = 0; v < V; ++v) {
        if (!((mask >> v) & 1u)) continue;
        double e2;
        robust_reproj2(u + 2 * v, P + 12 * v, x, e2);
        s2 += e2;
      }
      r = sqrt(s2 / robust_count(mask));
      ok = isfinite(r);
    }
  }
  if (red.lane != 0) return;
  for (int k = 0; k < 3; ++k) X[k] = ok ? x[k] : 0.0;
  *inl = ok ? (int32_t)mask : 0;
  *resid = ok ? r : 0.0;
  *status = ok ? 1 : 0;
}

// u [NT][V][J][stride_u], P [NT][V][12], w [NT][V][J] or null (ones); one warp per (tuple, joint),
// its views staged in shared memory (lanes >= V load no point, lanes stride over the V*12 entries of P)
constexpr int kRobustWarps = 4;

__global__ void __launch_bounds__(kRobustWarps * 32)
triangulate_robust_kernel(const double* __restrict__ u, int stride_u, const double* __restrict__ P,
                          const double* __restrict__ w, int NT, int V, int J, double thr,
                          double* __restrict__ X, int32_t* __restrict__ inl,
                          double* __restrict__ resid, int32_t* __restrict__ status) {
  __shared__ double sP[kRobustWarps][RB_MAXV * 12], sU[kRobustWarps][RB_MAXV * 2],
      sW[kRobustWarps][RB_MAXV];
  const int wid = threadIdx.x >> 5;
  const int64_t idx = (int64_t)blockIdx.x * kRobustWarps + wid;
  if (idx >= (int64_t)NT * J) return;                      // warp-uniform
  RbWarp red;
  red.lane = threadIdx.x & 31;
  const int64_t t = idx / J, j = idx - t * J;
  for (int k = red.lane; k < V * 12; k += 32) sP[wid][k] = P[t * V * 12 + k];
  if (red.lane < V) {
    const int64_t o = (t * V + red.lane) * J + j;
    sU[wid][2 * red.lane + 0] = u[o * stride_u + 0];
    sU[wid][2 * red.lane + 1] = u[o * stride_u + 1];
    sW[wid][red.lane] = w ? w[o] : 1.0;
  }
  __syncwarp();
  robust_point(red, sU[wid], sP[wid], sW[wid], V, thr, X + idx * 3, inl + idx, resid + idx,
               status + idx);
}

// --------------------------------------------------------------- tuple labels (online training)
// A view-major training batch: T tuples of V views, row v*T + t is view v of tuple t.
// 1. tuple_point: one (tuple t, joint j).  The lanes stage the V views in u [V*2], P [V*12], w [V]
//    (lane l: views l, l + n, ..; entries l, l + n, .. of P): the image point of row v*T + t with the
//    arithmetic of patch_to_image_kernel, its projection matrix, and its weight lse_ws[1] (the peak
//    softmax probability of the joint) or 1.  Then robust_point, as in triangulate_robust_kernel.
template <class Red>
__host__ __device__ void tuple_point(const Red& red, const float* coords, const float* lse_ws, const double* box,
                                     const double* P, int64_t T, int V, int J, int64_t t, int j, double patch_w,
                                     double patch_h, double rect3d_w, double thr, double* u, double* Pv,
                                     double* w, double* X, int32_t* inl, double* resid, int32_t* status) {
  for (int k = red.lane; k < V * 12; k += red.n) {
    const int v = k / 12;
    Pv[k] = P[(v * T + t) * 12 + (k - v * 12)];
  }
  for (int v = red.lane; v < V; v += red.n) {
    const int64_t o = (v * T + t) * J + j;
    double kp[4];
    patch_to_image_point(coords + o * 3, box + (v * T + t) * 6, patch_w, patch_h, rect3d_w, kp);
    u[2 * v + 0] = kp[0];
    u[2 * v + 1] = kp[1];
    w[v] = lse_ws ? (double)lse_ws[o * 2 + 1] : 1.0;
  }
#ifdef __CUDA_ARCH__
  __syncwarp();
#endif
  robust_point(red, u, Pv, w, V, thr, X, inl, resid, status);
}

// 2. tuple_label: one (row, joint).  X, status [T][J].  Label and weight 1 when the joint and the root
//    (joint 0) of the tuple were triangulated and both lie at a positive, finite depth in this view
//    (and the label is finite); label 0 and weight 0 otherwise.
__host__ __device__ inline void tuple_label(const double* X, const int32_t* status, const double* cam,
                                            const double* box, int64_t T, int J, int64_t row, int j, double patch_w,
                                            double patch_h, double rect3d_w, float* label, float* weight) {
  const int64_t t = row % T;
  const double* xt = X + t * J * 3;
  float lab[3];
  double cz, pz;
  project_label_point(xt + (int64_t)j * 3, xt, cam + row * 16, box + row * 6, patch_w, patch_h, rect3d_w, lab,
                      cz, pz);
  const bool ok = status[t * J + j] == 1 && status[t * J] == 1 && cz > 0.0 && cz < INFINITY && pz > 0.0 &&
                  pz < INFINITY && isfinite(lab[0]) && isfinite(lab[1]) && isfinite(lab[2]);
  for (int k = 0; k < 3; ++k) {
    label[k] = ok ? lab[k] : 0.f;
    weight[k] = ok ? 1.f : 0.f;
  }
}

__global__ void __launch_bounds__(kRobustWarps * 32)
tuple_triangulate_kernel(const float* __restrict__ coords, const float* __restrict__ lse_ws,
                         const double* __restrict__ box, const double* __restrict__ P, int T, int V, int J,
                         double patch_w, double patch_h, double rect3d_w, double thr, double* __restrict__ X,
                         int32_t* __restrict__ inl, double* __restrict__ resid, int32_t* __restrict__ status) {
  __shared__ double sP[kRobustWarps][RB_MAXV * 12], sU[kRobustWarps][RB_MAXV * 2],
      sW[kRobustWarps][RB_MAXV];
  const int wid = threadIdx.x >> 5;
  const int64_t idx = (int64_t)blockIdx.x * kRobustWarps + wid;
  if (idx >= (int64_t)T * J) return;                       // warp-uniform
  RbWarp red;
  red.lane = threadIdx.x & 31;
  const int64_t t = idx / J;
  const int j = (int)(idx - t * J);
  tuple_point(red, coords, lse_ws, box, P, T, V, J, t, j, patch_w, patch_h, rect3d_w, thr, sU[wid], sP[wid],
              sW[wid], X + idx * 3, inl + idx, resid + idx, status + idx);
}

__global__ void tuple_label_kernel(const double* __restrict__ X, const int32_t* __restrict__ status,
                                   const double* __restrict__ cam, const double* __restrict__ box, int T, int V,
                                   int J, double patch_w, double patch_h, double rect3d_w,
                                   float* __restrict__ label, float* __restrict__ weight) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)V * T * J) return;
  const int64_t row = idx / J;
  tuple_label(X, status, cam, box, T, J, row, (int)(idx - row * J), patch_w, patch_h, rect3d_w, label + idx * 3,
              weight + idx * 3);
}

// --------------------------------------------------------------- argmax
// inference.py:24-39: one warp per (n,j) map; (value, index) reduction with
// smallest-index tie-break == numpy argmax first-occurrence.  NaN: numpy
// treats the first NaN as the maximum; reproduced by ordering NaN above all.
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) {
  const bool vn = (v != v), bn = (bv != bv);
  if (vn || bn) return vn && (!bn || i < bi);
  return v > bv || (v == bv && i < bi);
}

__global__ void argmax2d_kernel(const float* __restrict__ hm, int NJ, int HW, int W,
                                int32_t* __restrict__ idx_out, float* __restrict__ maxval,
                                float* __restrict__ preds) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= NJ) return;
  const float* p = hm + (int64_t)warp * HW;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = lane; i < HW; i += 32) {
    const float v = p[i];
    if (better(v, i, bv, bi)) { bv = v; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  if (lane == 0) {
    if (bi == 0x7fffffff) bi = 0;  // all -inf: numpy returns index 0
    if (idx_out) idx_out[warp] = bi;
    if (maxval) maxval[warp] = bv;
    if (preds) {
      const float mask = (bv > 0.f) ? 1.f : 0.f;   // :35-39
      preds[warp * 2 + 0] = (float)(bi % W) * mask;
      preds[warp * 2 + 1] = floorf((float)bi / (float)W) * mask;
    }
  }
}

}  // namespace

extern "C" __attribute__((visibility("default"))) int epb_triangulate(const double* u1, const double* u2, int stride_u, const double* P1,
                               const double* P2, int NP, int J, int method, double tol, double* X,
                               int32_t* status, epb_stream_t stream) {
  EPB_CHECK_ARG(u1 && u2 && P1 && P2 && X);
  EPB_CHECK_ARG(NP >= 0 && J >= 0 && stride_u >= 2);
  EPB_CHECK_ARG(method >= 0 && method <= 4);
  if (NP * J == 0) return EPB_OK;
  const int n = NP * J;
  cudaStream_t st = as_stream(stream);
  double* Fpair = nullptr;
  if (method >= 3) {
    // one fundamental matrix per pair (from the projection matrices, or the 8-point fallback)
    int rc = epb_workspace(EPB_WS_FPAIR, (size_t)NP * 9 * sizeof(double), st, (void**)&Fpair);
    if (rc) return rc;
    pair_fundamental_kernel<<<(NP + 63) / 64, 64, 0, st>>>(u1, u2, stride_u, P1, P2, NP, J, method,
                                                           Fpair);
    EPB_LAUNCH_CHECK();
  }
  triangulate_kernel<<<(n + 63) / 64, 64, 0, st>>>(u1, u2, stride_u, P1, P2, NP, J, method, tol,
                                                   Fpair, X, status);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_relative_pose(
    const double* u, int stride_u, const double* intr, const double* box, int B, int J,
    double rect3d_w, double* Pa, double* Pb, double* cam, int32_t* inliers, int32_t* status,
    int32_t* diag, epb_stream_t stream) {
  EPB_CHECK_ARG(u && intr && box && Pa && Pb && cam && inliers && status);
  EPB_CHECK_ARG(B >= 0 && B % 2 == 0 && J >= 8 && J <= RP_MAXJ && stride_u >= 2);
  const int NP = B / 2;
  if (NP == 0) return EPB_OK;
  const int threads = 128;                         // 4 pairs per block, one warp each
  relative_pose_kernel<<<(NP * 32 + threads - 1) / threads, threads, 0, as_stream(stream)>>>(
      u, stride_u, intr, box, NP, J, rect3d_w, Pa, Pb, cam, inliers, status, diag);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_patch_to_image(const float* coords, const double* box, int B, int J,
                                  double patch_w, double patch_h, double rect3d_w, double* kps,
                                  epb_stream_t stream) {
  EPB_CHECK_ARG(coords && box && kps);
  EPB_CHECK_ARG(B >= 0 && J >= 0);
  if (B * J == 0) return EPB_OK;
  const int n = B * J;
  patch_to_image_kernel<<<(n + 127) / 128, 128, 0, as_stream(stream)>>>(coords, box, B, J, patch_w,
                                                                       patch_h, rect3d_w, kps);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_project_labels(const double* X, const double* cam, const double* box, int B,
                                  int J, double patch_w, double patch_h, double rect3d_w,
                                  float* label, float* weight, epb_stream_t stream) {
  EPB_CHECK_ARG(X && cam && box && label && weight);
  EPB_CHECK_ARG(B >= 0 && J >= 0);
  if (B * J == 0) return EPB_OK;
  const int n = B * J;
  project_labels_kernel<<<(n + 127) / 128, 128, 0, as_stream(stream)>>>(
      X, cam, box, B, J, patch_w, patch_h, rect3d_w, label, weight);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_argmax2d(const float* hm, int NJ, int H, int W, int32_t* idx, float* maxval,
                            float* preds, epb_stream_t stream) {
  EPB_CHECK_ARG(hm && NJ >= 0 && H > 0 && W > 0);
  if (NJ == 0) return EPB_OK;
  const int threads = 256;
  const int blocks = (NJ * 32 + threads - 1) / threads;
  argmax2d_kernel<<<blocks, threads, 0, as_stream(stream)>>>(hm, NJ, H * W, W, idx, maxval, preds);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_h36m_eval(
    const double* pred, const double* gt, const double* cam, int S, int J, int root,
    uint32_t j14mask, double pck_thr, double* metrics, double* per_joint, int32_t* pck,
    double* poses, epb_stream_t stream) {
  EPB_CHECK_ARG(pred && gt && cam && metrics);
  EPB_CHECK_ARG(S >= 0 && J > 0 && J <= 32 && root >= 0 && root < J);
  if (S == 0) return EPB_OK;
  h36m_eval_kernel<<<(S + 63) / 64, 64, 0, as_stream(stream)>>>(pred, gt, cam, S, J, root, j14mask,
                                                               pck_thr, metrics, per_joint, pck,
                                                               poses);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_pose_errors(
    const double* pred, const double* gt, int S, int J, uint32_t submask, double* metrics, double* per_joint,
    epb_stream_t stream) {
  EPB_CHECK_ARG(pred && gt && metrics);
  EPB_CHECK_ARG(S >= 0 && J > 0 && J <= 32);
  if (S == 0) return EPB_OK;
  pose_errors_kernel<<<(S + 63) / 64, 64, 0, as_stream(stream)>>>(pred, gt, S, J, submask, metrics, per_joint);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_pose_to_camera(
    const double* joints, const double* cam, int N, int J, int root, double* out, epb_stream_t stream) {
  EPB_CHECK_ARG(joints && cam && out);
  EPB_CHECK_ARG(N >= 0 && J > 0 && root >= 0 && root < J);
  if (N == 0) return EPB_OK;
  pose_to_camera_kernel<<<(N + 63) / 64, 64, 0, as_stream(stream)>>>(joints, cam, N, J, root, out);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_pseudo_records(
    const double* X, const int32_t* status, const double* cam, int T, int S, int V, int J, int root, double* joints_3d,
    double* vis, double* pelvis, int32_t* ok, epb_stream_t stream) {
  EPB_CHECK_ARG(X && status && cam && joints_3d && vis && pelvis && ok);
  const int rc = pseudo_records_sizes(T, S, V, J, root);
  if (rc != EPB_OK) return rc;
  if (T == 0) return EPB_OK;
  const int threads = 128;
  const int64_t n = (int64_t)T * V;
  pseudo_records_kernel<<<(unsigned)((n + threads - 1) / threads), threads, 0, as_stream(stream)>>>(
      X, status, cam, T, S, V, J, root, joints_3d, vis, pelvis, ok);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_triangulate_nview(
    const double* u, int stride_u, const double* P, int NT, int V, int J, double* X, int32_t* status,
    epb_stream_t stream) {
  EPB_CHECK_ARG(u && P && X);
  EPB_CHECK_ARG(NT >= 0 && J >= 0 && stride_u >= 2 && V >= 2 && V <= 4);
  if (NT * J == 0) return EPB_OK;
  const int n = NT * J;
  triangulate_nview_kernel<<<(n + 63) / 64, 64, 0, as_stream(stream)>>>(u, stride_u, P, NT, V, J, X, status);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_triangulate_robust(
    const double* u, int stride_u, const double* P, const double* w, int NT, int V, int J,
    double threshold_px, double* X, int32_t* inliers, double* resid, int32_t* status,
    epb_stream_t stream) {
  EPB_CHECK_ARG(u && P && X && inliers && resid && status);
  EPB_CHECK_ARG(NT >= 0 && J >= 0 && stride_u >= 2 && V >= 2 && V <= RB_MAXV);
  EPB_CHECK_ARG(isfinite(threshold_px) && threshold_px > 0.0);
  EPB_CHECK_ARG((int64_t)NT * J <= 0x7fffffff);
  if ((int64_t)NT * J == 0) return EPB_OK;
  const int64_t n = (int64_t)NT * J;
  triangulate_robust_kernel<<<(unsigned)((n + kRobustWarps - 1) / kRobustWarps), kRobustWarps * 32, 0,
                              as_stream(stream)>>>(u, stride_u, P, w, NT, V, J, threshold_px, X,
                                                   inliers, resid, status);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_tuple_labels(
    const float* coords, const float* lse_ws, const double* box, const double* P, const double* cam, int T,
    int V, int J, double patch_w, double patch_h, double rect3d_w, double threshold_px, float* label,
    float* weight, double* X, int32_t* inliers, double* resid, int32_t* status, epb_stream_t stream) {
  EPB_CHECK_ARG(coords && box && P && cam && label && weight && X && inliers && resid && status);
  EPB_CHECK_ARG(T >= 0 && J >= 0 && V >= 2 && V <= RB_MAXV);
  EPB_CHECK_ARG(isfinite(threshold_px) && threshold_px > 0.0);
  EPB_CHECK_ARG((int64_t)V * T * J <= 0x7fffffff);
  if ((int64_t)T * J == 0) return EPB_OK;
  cudaStream_t st = as_stream(stream);
  const int64_t n = (int64_t)T * J;
  tuple_triangulate_kernel<<<(unsigned)((n + kRobustWarps - 1) / kRobustWarps), kRobustWarps * 32, 0, st>>>(
      coords, lse_ws, box, P, T, V, J, patch_w, patch_h, rect3d_w, threshold_px, X, inliers, resid, status);
  EPB_LAUNCH_CHECK();
  const int64_t m = (int64_t)V * T * J;
  tuple_label_kernel<<<(unsigned)((m + 127) / 128), 128, 0, st>>>(X, status, cam, box, T, V, J, patch_w, patch_h,
                                                                  rect3d_w, label, weight);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}
