// eig3.cuh — symmetric 3x3 eigen-decomposition in float64 for the normal/planarity kernel.
//
// Reference: np.linalg.eig on np.cov output (python/simpleicp/pointcloud.py:190-198).  NumPy
// calls LAPACK dgeev, whose eigenvector SIGN is an artefact of its algorithm (no geometric
// meaning) but decides the sign of every point-to-plane distance downstream (median / MAD,
// corrpts.py:184-187).  `eig3_dgeev` therefore follows dgeev's published algorithm for a 3 x 3
// input step by step — dgebal('B') (its scaling is a no-op for symmetric input, its permutation
// is not: a row whose off-diagonal entries are exactly zero, as on an axis-aligned wall, is
// isolated and moved to the end), dgehd2 (one Householder reflector) and dorghr on the remaining
// block, dlahqr (double-shift QR with the Ahues-Tisseur deflation test, dlanv2 for the final
// 2 x 2 block), dtrevc back-substitution and back-transformation, max-norm scaling, dgebak's row
// swap, 2-norm scaling — so that eigenvalue slots and eigenvector signs come out as NumPy's do.
// Measured agreement with np.linalg.eig on 12 000 neighbourhood covariances of the reference's
// data sets: 99.8 %; the rest are inputs whose deflation test sits within rounding of its
// threshold (one QR sweep more or fewer flips two columns).  On designed covariances (exact zero
// off-diagonals, rank 0 and 1, repeated eigenvalues) the float32 normals are bit-identical
// (tests/test_eig3_host.py).  `eig3_jacobi` (cyclic Jacobi, canonical sign) is the other mode.
//
// Header-only and compilable by a host C++ compiler (tests build it with g++ and compare with
// NumPy on the CPU).
#pragma once
#include <math.h>

#include "../../include/sicp_b200.h"

#ifndef __CUDACC__
#ifndef __host__
#define __host__
#endif
#ifndef __device__
#define __device__
#endif
#endif

namespace sicp {

// Cyclic Jacobi on a symmetric 3x3 matrix.  a is destroyed (its diagonal becomes the
// eigenvalues), v receives the eigenvectors as columns.
__host__ __device__ inline void eig3_jacobi(double a[3][3], double v[3][3]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) v[i][j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 64; ++sweep) {
    const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
    const double dia = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2];
    if (off <= 1e-34 * dia || off == 0.0) break;
    for (int p = 0; p < 2; ++p) {
      for (int q = p + 1; q < 3; ++q) {
        const double apq = a[p][q];
        if (apq == 0.0) continue;
        const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
        double t;
        if (fabs(theta) > 1e150) {
          t = 0.5 / theta;
        } else {
          t = 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
          if (theta < 0.0) t = -t;
        }
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        const int r = 3 - p - q;  // the third index
        const double app = a[p][p], aqq = a[q][q];
        a[p][p] = app - t * apq;
        a[q][q] = aqq + t * apq;
        a[p][q] = a[q][p] = 0.0;
        const double arp = a[r][p], arq = a[r][q];
        a[r][p] = a[p][r] = c * arp - s * arq;
        a[r][q] = a[q][r] = s * arp + c * arq;
        for (int i = 0; i < 3; ++i) {
          const double vip = v[i][p], viq = v[i][q];
          v[i][p] = c * vip - s * viq;
          v[i][q] = s * vip + c * viq;
        }
      }
    }
  }
}

namespace dgeev3 {

constexpr double kEps = 2.220446049250313e-16;      // dlamch('P')
constexpr double kSafmin = 2.2250738585072014e-308;  // dlamch('S')

__host__ __device__ inline double sgn(double a, double b) { return (b >= 0.0) ? fabs(a) : -fabs(a); }

__host__ __device__ inline void swap2(double& a, double& b) {
  const double t = a;
  a = b;
  b = t;
}

__host__ __device__ inline double lapy2(double x, double y) {
  const double w = fmax(fabs(x), fabs(y)), z = fmin(fabs(x), fabs(y));
  if (z == 0.0) return w;
  const double q = z / w;
  return w * sqrt(1.0 + q * q);
}

// dlarfg for n = 2 or 3: alpha in/out (beta), x[0..n-2] in/out (v(2:)), returns tau.
__host__ __device__ inline double larfg(int n, double& alpha, double* x) {
  const double xnorm = (n == 3) ? hypot(x[0], x[1]) : fabs(x[0]);
  if (xnorm == 0.0) return 0.0;
  const double beta = -sgn(lapy2(alpha, xnorm), alpha);
  const double tau = (beta - alpha) / beta;
  const double scal = 1.0 / (alpha - beta);
  for (int i = 0; i < n - 1; ++i) x[i] *= scal;
  alpha = beta;
  return tau;
}

// dlanv2: Schur factorisation of a real 2 x 2 block in standard form.
__host__ __device__ inline void lanv2(double& a, double& b, double& c, double& d, double& cs, double& sn) {
  const double multpl = 4.0;
  if (c == 0.0) {
    cs = 1.0;
    sn = 0.0;
  } else if (b == 0.0) {
    cs = 0.0;
    sn = 1.0;
    const double temp = d;
    d = a;
    a = temp;
    b = -c;
    c = 0.0;
  } else if ((a - d) == 0.0 && sgn(1.0, b) != sgn(1.0, c)) {
    cs = 1.0;
    sn = 0.0;
  } else {
    double temp = a - d;
    double p = 0.5 * temp;
    const double bcmax = fmax(fabs(b), fabs(c));
    const double bcmis = fmin(fabs(b), fabs(c)) * sgn(1.0, b) * sgn(1.0, c);
    const double scale = fmax(fabs(p), bcmax);
    double z = (p / scale) * p + (bcmax / scale) * bcmis;
    if (z >= multpl * kEps) {
      z = p + sgn(sqrt(scale) * sqrt(z), p);
      a = d + z;
      d = d - (bcmax / z) * bcmis;
      const double tau = lapy2(c, z);
      cs = z / tau;
      sn = c / tau;
      b = b - c;
      c = 0.0;
    } else {
      const double sigma = b + c;
      double tau = lapy2(sigma, temp);
      cs = sqrt(0.5 * (1.0 + fabs(sigma) / tau));
      sn = -(p / (tau * cs)) * sgn(1.0, sigma);
      const double aa = a * cs + b * sn, bb = -a * sn + b * cs;
      const double cc = c * cs + d * sn, dd = -c * sn + d * cs;
      a = aa * cs + cc * sn;
      b = bb * cs + dd * sn;
      c = -aa * sn + cc * cs;
      d = -bb * sn + dd * cs;
      temp = 0.5 * (a + d);
      a = temp;
      d = temp;
      if (c != 0.0) {
        if (b != 0.0) {
          if (sgn(1.0, b) == sgn(1.0, c)) {
            const double sab = sqrt(fabs(b)), sac = sqrt(fabs(c));
            p = sgn(sab * sac, c);
            tau = 1.0 / sqrt(fabs(b + c));
            a = temp + p;
            d = temp - p;
            b = b - c;
            c = 0.0;
            const double cs1 = sab * tau, sn1 = sac * tau;
            temp = cs * cs1 - sn * sn1;
            sn = cs * sn1 + sn * cs1;
            cs = temp;
          }
        } else {
          b = -c;
          c = 0.0;
          temp = cs;
          cs = -sn;
          sn = temp;
        }
      }
    }
  }
}

}  // namespace dgeev3

namespace dgeev3 {

// dgeev after dgebal's permutation: h = P A P^T, QR on rows/columns 0..IHI (a template
// parameter, so that the full 3 x 3 path carries no block bounds in registers); dgebak swaps the
// eigenvector rows piv <-> 2 back.
template <int IHI>
__host__ __device__ inline bool dgeev_core(double h[3][3], int piv, double wr[3], double vr[3][3]) {
  double z[3][3];
  // dgehd2 on ilo..ihi: one reflector acting on rows/columns 1..2 (the identity unless IHI = 2)
  z[0][0] = 1.0; z[0][1] = 0.0; z[0][2] = 0.0;
  z[1][0] = 0.0; z[1][1] = 1.0; z[1][2] = 0.0;
  z[2][0] = 0.0; z[2][1] = 0.0; z[2][2] = 1.0;
  if (IHI == 2) {
    double v1[2];
    double alpha = h[1][0];
    double x[1] = {h[2][0]};
    const double tau = larfg(2, alpha, x);
    v1[0] = 1.0;
    v1[1] = x[0];
    h[1][0] = alpha;
    h[2][0] = 0.0;
    for (int i = 0; i < 3; ++i) {
      const double s = h[i][1] * v1[0] + h[i][2] * v1[1];
      h[i][1] -= tau * s * v1[0];
      h[i][2] -= tau * s * v1[1];
    }
    for (int j = 1; j < 3; ++j) {
      const double s = v1[0] * h[1][j] + v1[1] * h[2][j];
      h[1][j] -= tau * s * v1[0];
      h[2][j] -= tau * s * v1[1];
    }
    // dorghr
    z[1][1] = 1.0 - tau * v1[0] * v1[0]; z[1][2] = -tau * v1[0] * v1[1];
    z[2][1] = -tau * v1[1] * v1[0]; z[2][2] = 1.0 - tau * v1[1] * v1[1];
  }
  // dhseqr: the eigenvalues dgebal isolated
  if (IHI < 2) wr[2] = h[2][2];
  if (IHI < 1) wr[1] = h[1][1];
  // dlahqr (ilo = 0, ihi = IHI, wantt, wantz with iloz = ilo, ihiz = ihi)
  const int ilo = 0, ihi = IHI, i1 = 0, i2 = 2;
  const double ulp = kEps, smlnum = kSafmin * ((double)(ihi - ilo + 1) / kEps);
  const int itmax = 300;
  int kdefl = 0;
  int i = ihi;
  while (i >= ilo) {
    int l = ilo;
    bool converged = false;
    for (int its = 0; its <= itmax; ++its) {
      int k = i;
      for (; k > l; --k) {
        if (fabs(h[k][k - 1]) <= smlnum) break;
        double tst = fabs(h[k - 1][k - 1]) + fabs(h[k][k]);
        if (tst == 0.0) {
          if (k - 2 >= ilo) tst += fabs(h[k - 1][k - 2]);
          if (k + 1 <= ihi) tst += fabs(h[k + 1][k]);
        }
        if (fabs(h[k][k - 1]) <= ulp * tst) {
          const double ab = fmax(fabs(h[k][k - 1]), fabs(h[k - 1][k]));
          const double ba = fmin(fabs(h[k][k - 1]), fabs(h[k - 1][k]));
          const double aa = fmax(fabs(h[k][k]), fabs(h[k - 1][k - 1] - h[k][k]));
          const double bb = fmin(fabs(h[k][k]), fabs(h[k - 1][k - 1] - h[k][k]));
          const double s = aa + ab;
          if (ba * (ab / s) <= fmax(smlnum, ulp * (bb * (aa / s)))) break;
        }
      }
      l = k;
      if (l > ilo) h[l][l - 1] = 0.0;
      if (l >= i - 1) {
        converged = true;
        break;
      }
      ++kdefl;
      double h11, h12, h21, h22;
      if (kdefl % 20 == 0) {
        const double s = fabs(h[i][i - 1]) + fabs(h[i - 1][i - 2]);
        h11 = 0.75 * s + h[i][i]; h12 = -0.4375 * s; h21 = s; h22 = h11;
      } else if (kdefl % 10 == 0) {
        const double s = fabs(h[l + 1][l]) + fabs(h[l + 2][l + 1]);
        h11 = 0.75 * s + h[l][l]; h12 = -0.4375 * s; h21 = s; h22 = h11;
      } else {
        h11 = h[i - 1][i - 1]; h21 = h[i][i - 1]; h12 = h[i - 1][i]; h22 = h[i][i];
      }
      double rt1r, rt1i, rt2r, rt2i;
      double s = fabs(h11) + fabs(h12) + fabs(h21) + fabs(h22);
      if (s == 0.0) {
        rt1r = rt1i = rt2r = rt2i = 0.0;
      } else {
        h11 /= s; h21 /= s; h12 /= s; h22 /= s;
        const double tr = (h11 + h22) / 2.0;
        const double det = (h11 - tr) * (h22 - tr) - h12 * h21;
        const double rtdisc = sqrt(fabs(det));
        if (det >= 0.0) {
          rt1r = tr * s; rt2r = rt1r; rt1i = rtdisc * s; rt2i = -rt1i;
        } else {
          rt1r = tr + rtdisc; rt2r = tr - rtdisc;
          if (fabs(rt1r - h22) <= fabs(rt2r - h22)) {
            rt1r = rt1r * s; rt2r = rt1r;
          } else {
            rt2r = rt2r * s; rt1r = rt2r;
          }
          rt1i = rt2i = 0.0;
        }
      }
      // the active block is the whole 3 x 3 here (l = 0, i = 2): m = i - 2 = l
      const int m = i - 2;
      double v[3];
      {
        double h21s = fabs(h[m + 1][m]);
        double ss = fabs(h[m][m] - rt2r) + fabs(rt2i) + h21s;
        h21s = h[m + 1][m] / ss;
        v[0] = h21s * h[m][m + 1] + (h[m][m] - rt1r) * ((h[m][m] - rt2r) / ss) - rt1i * (rt2i / ss);
        v[1] = h21s * (h[m][m] + h[m + 1][m + 1] - rt1r - rt2r);
        v[2] = h21s * h[m + 2][m + 1];
        ss = fabs(v[0]) + fabs(v[1]) + fabs(v[2]);
        v[0] /= ss; v[1] /= ss; v[2] /= ss;
      }
      for (int kk = m; kk < i; ++kk) {
        const int nr = (i - kk + 1 < 3) ? (i - kk + 1) : 3;
        if (kk > m)
          for (int t = 0; t < nr; ++t) v[t] = h[kk + t][kk - 1];
        const double t1 = larfg(nr, v[0], &v[1]);
        if (kk > m) {
          h[kk][kk - 1] = v[0];
          h[kk + 1][kk - 1] = 0.0;
          if (kk < i - 1) h[kk + 2][kk - 1] = 0.0;
        } else if (m > l) {
          h[kk][kk - 1] = h[kk][kk - 1] * (1.0 - t1);
        }
        const double v2 = v[1], t2 = t1 * v2;
        if (nr == 3) {
          const double v3 = v[2], t3 = t1 * v3;
          for (int j = kk; j <= i2; ++j) {
            const double sm = h[kk][j] + v2 * h[kk + 1][j] + v3 * h[kk + 2][j];
            h[kk][j] -= sm * t1; h[kk + 1][j] -= sm * t2; h[kk + 2][j] -= sm * t3;
          }
          const int jmax = (kk + 3 < i) ? kk + 3 : i;
          for (int j = i1; j <= jmax; ++j) {
            const double sm = h[j][kk] + v2 * h[j][kk + 1] + v3 * h[j][kk + 2];
            h[j][kk] -= sm * t1; h[j][kk + 1] -= sm * t2; h[j][kk + 2] -= sm * t3;
          }
          for (int j = 0; j < 3; ++j) {
            const double sm = z[j][kk] + v2 * z[j][kk + 1] + v3 * z[j][kk + 2];
            z[j][kk] -= sm * t1; z[j][kk + 1] -= sm * t2; z[j][kk + 2] -= sm * t3;
          }
        } else {
          for (int j = kk; j <= i2; ++j) {
            const double sm = h[kk][j] + v2 * h[kk + 1][j];
            h[kk][j] -= sm * t1; h[kk + 1][j] -= sm * t2;
          }
          for (int j = i1; j <= i; ++j) {
            const double sm = h[j][kk] + v2 * h[j][kk + 1];
            h[j][kk] -= sm * t1; h[j][kk + 1] -= sm * t2;
          }
          for (int j = 0; j < 3; ++j) {
            const double sm = z[j][kk] + v2 * z[j][kk + 1];
            z[j][kk] -= sm * t1; z[j][kk + 1] -= sm * t2;
          }
        }
      }
    }
    if (!converged) return false;
    if (l == i) {
      wr[i] = h[i][i];
    } else {
      double cs, sn;
      lanv2(h[i - 1][i - 1], h[i - 1][i], h[i][i - 1], h[i][i], cs, sn);
      wr[i - 1] = h[i - 1][i - 1];
      wr[i] = h[i][i];
      for (int j = i + 1; j <= i2; ++j) {
        const double t = cs * h[i - 1][j] + sn * h[i][j];
        h[i][j] = cs * h[i][j] - sn * h[i - 1][j];
        h[i - 1][j] = t;
      }
      for (int j = i1; j < i - 1; ++j) {
        const double t = cs * h[j][i - 1] + sn * h[j][i];
        h[j][i] = cs * h[j][i] - sn * h[j][i - 1];
        h[j][i - 1] = t;
      }
      for (int j = ilo; j <= ihi; ++j) {
        const double t = cs * z[j][i - 1] + sn * z[j][i];
        z[j][i] = cs * z[j][i] - sn * z[j][i - 1];
        z[j][i - 1] = t;
      }
    }
    kdefl = 0;
    i = l - 1;
  }
  // dtrevc: back-substitution on the (quasi) triangular T = h, back-transform with Z, scale
  for (int ki = 2; ki >= 0; --ki) {
    double x[3] = {0.0, 0.0, 0.0}, work[3] = {0.0, 0.0, 0.0};
    x[ki] = 1.0;
    for (int j = 0; j < ki; ++j) work[j] = -h[j][ki];
    const double smin = fmax(kEps * fabs(wr[ki]), kSafmin * 3.0 / kEps);
    for (int j = ki - 1; j >= 0; --j) {
      double den = h[j][j] - wr[ki];
      if (fabs(den) < smin) den = smin;
      const double xj = work[j] / den;
      x[j] = xj;
      for (int t = 0; t < j; ++t) work[t] -= xj * h[t][j];
    }
    double col[3];
    for (int r = 0; r < 3; ++r) {
      double acc = 0.0;
      for (int c = 0; c <= ki; ++c) acc += z[r][c] * x[c];
      col[r] = acc;
    }
    const double emax = fmax(fabs(col[0]), fmax(fabs(col[1]), fabs(col[2])));
    for (int r = 0; r < 3; ++r) col[r] /= emax;
    // dgebak: undo dgebal's row swap before dgeev's 2-norm scaling
    if (IHI < 2 && piv == 0) swap2(col[0], col[2]);
    if (IHI < 2 && piv == 1) swap2(col[1], col[2]);
    const double nrm = sqrt(col[0] * col[0] + col[1] * col[1] + col[2] * col[2]);
    for (int r = 0; r < 3; ++r) vr[r][ki] = col[r] / nrm;
  }
  return true;
}

// The rare blocks after an isolation, out of line: the common full-block path keeps its registers.
#ifdef __CUDACC__
__noinline__
#endif
static __host__ __device__ bool dgeev_isolated(double h[3][3], int ihi, int piv, double wr[3], double vr[3][3]) {
  return (ihi == 1) ? dgeev_core<1>(h, piv, wr, vr) : dgeev_core<0>(h, piv, wr, vr);
}

}  // namespace dgeev3

// dgeev on a symmetric 3 x 3 matrix: wr = eigenvalues in LAPACK's slot order, vr = unit
// eigenvectors as columns with LAPACK's signs.  Returns false if the QR iteration fails.
__host__ __device__ inline bool eig3_dgeev(const double A[3][3], double wr[3], double vr[3][3]) {
  using namespace dgeev3;
  double h[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) h[i][j] = A[i][j];
  // dgebal('B'), permutation phase.  The row search (from the last row up, pushing a row whose
  // off-diagonal entries within the active block are all exactly zero to the block's end) on a
  // symmetric 3 x 3 input: row 2 isolated stays (and with c01 = 0 too, rows 1 and 0 follow in place:
  // ilo = ihi = 0); else row 1 or row 0 isolated is swapped with row 2.  The column search then
  // finds nothing: a column isolated in a symmetric block is an isolated row the search would
  // have taken.  The scaling phase is a no-op (row and column norms are equal).  So P A P^T swaps
  // `piv` with 2 (or nothing), QR runs on 0..ihi, and dgebak swaps the eigenvector rows back.
  int ihi = 2, piv = 2;
  if (h[2][0] == 0.0 && h[2][1] == 0.0) {
    ihi = (h[1][0] == 0.0) ? 0 : 1;
  } else if ((h[1][0] == 0.0 && h[1][2] == 0.0) || (h[0][1] == 0.0 && h[0][2] == 0.0)) {
    piv = (h[1][0] == 0.0 && h[1][2] == 0.0) ? 1 : 0;
    ihi = 1;
    // columns piv <-> 2, then rows piv <-> 2, written out (constant indices keep h in registers)
    if (piv == 0) {
      swap2(h[0][0], h[2][2]); swap2(h[0][1], h[2][1]); swap2(h[0][2], h[2][0]); swap2(h[1][0], h[1][2]);
    } else {
      swap2(h[1][1], h[2][2]); swap2(h[0][1], h[0][2]); swap2(h[1][0], h[2][0]); swap2(h[1][2], h[2][1]);
    }
  }
  switch (ihi) {
    case 2: return dgeev_core<2>(h, piv, wr, vr);
    default: return dgeev3::dgeev_isolated(h, ihi, piv, wr, vr);
  }
}

// Eigenvalues sorted descending in w; n = unit eigenvector of the smallest eigenvalue.
// sign_mode SICP_SIGN_DGEEV: NumPy / LAPACK sign; SICP_SIGN_CANONICAL: largest component > 0.
__host__ __device__ inline void eig3_smallest(double c00, double c01, double c02, double c11,
                                              double c12, double c22, int sign_mode, double w[3],
                                              double n[3]) {
  const double scale =
      fmax(fmax(fabs(c00), fabs(c11)), fmax(fabs(c22), fmax(fabs(c01), fmax(fabs(c02), fabs(c12)))));
  if (!(scale > 0.0) || !isfinite(scale)) {
    // degenerate neighbourhood (all points coincide) or non-finite input: the reference's
    // planarity is 0/0 = NaN, which every rejection test drops.
    w[0] = w[1] = w[2] = (scale == 0.0) ? 0.0 : scale;
    n[0] = 1.0;
    n[1] = n[2] = 0.0;
    return;
  }
  if (sign_mode == SICP_SIGN_DGEEV) {
    const double A[3][3] = {{c00, c01, c02}, {c01, c11, c12}, {c02, c12, c22}};
    double wr[3], vr[3][3];
    if (eig3_dgeev(A, wr, vr)) {
      // reference: idx = eig_vals.argsort()[::-1] (pointcloud.py:192).  NumPy's argsort keeps
      // equal values in slot order at n = 3, so after the reversal the order is descending in
      // (value, slot): among equal eigenvalues the LOWEST slot comes last and is the normal.
      int i0 = 0, i1 = 1, i2 = 2;
      auto after = [&](int a, int b) { return wr[a] < wr[b] || (wr[a] == wr[b] && a < b); };
      if (after(i0, i1)) { const int t = i0; i0 = i1; i1 = t; }
      if (after(i1, i2)) { const int t = i1; i1 = i2; i2 = t; }
      if (after(i0, i1)) { const int t = i0; i0 = i1; i1 = t; }
      w[0] = wr[i0];
      w[1] = wr[i1];
      w[2] = wr[i2];
      n[0] = vr[0][i2];
      n[1] = vr[1][i2];
      n[2] = vr[2][i2];
      return;
    }
  }
  const double is = 1.0 / scale;
  double a[3][3] = {{c00 * is, c01 * is, c02 * is}, {c01 * is, c11 * is, c12 * is}, {c02 * is, c12 * is, c22 * is}};
  double v[3][3];
  eig3_jacobi(a, v);
  int i0 = 0, i1 = 1, i2 = 2;  // descending order of a[i][i]
  if (a[i0][i0] < a[i1][i1]) { const int t = i0; i0 = i1; i1 = t; }
  if (a[i1][i1] < a[i2][i2]) { const int t = i1; i1 = i2; i2 = t; }
  if (a[i0][i0] < a[i1][i1]) { const int t = i0; i0 = i1; i1 = t; }
  w[0] = a[i0][i0] * scale;
  w[1] = a[i1][i1] * scale;
  w[2] = a[i2][i2] * scale;
  double x = v[0][i2], y = v[1][i2], z = v[2][i2];
  const double nn = 1.0 / sqrt(x * x + y * y + z * z);
  x *= nn;
  y *= nn;
  z *= nn;
  // canonical sign: the component of largest magnitude is positive
  const double ax = fabs(x), ay = fabs(y), az = fabs(z);
  const double lead = (ax >= ay && ax >= az) ? x : ((ay >= az) ? y : z);
  if (lead < 0.0) {
    x = -x;
    y = -y;
    z = -z;
  }
  n[0] = x;
  n[1] = y;
  n[2] = z;
}

}  // namespace sicp
