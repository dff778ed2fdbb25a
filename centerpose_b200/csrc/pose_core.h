// Per-detection double-precision math of the CenterPose post-network path,
// written once as __host__ __device__ code: the CUDA decode kernel calls it
// per thread, and tests/ compile the same header with g++ to check it on the
// CPU against the oracle (no GPU needed for the math itself).
//
// Reference behaviour reproduced (paths relative to /root/reference/src/lib):
//   utils/pnp/cuboid_objectron.py:83-109   cuboid vertices, float32 arithmetic
//   utils/pnp/cuboid_pnp_solver.py:143-239 point filtering, cv2.solvePnPGeneric(ITERATIVE),
//                                          OpenCV -> OpenGL frame change, z < 0 failure
//   utils/pnp/cuboid_pnp_shell.py:24-93    kps_3d_cam, kps_pnp, visibility gates
//   detectors/object_pose.py:27-124        soft_nms_nvidia(method=2)
//   utils/gpfit.py:13-26                   moments()
// OpenCV's SOLVEPNP_ITERATIVE (third party, see oracle/pnp_ref.py header) =
// DLT start + Levenberg-Marquardt to the local least-squares minimum.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define CP_HD __host__ __device__ __forceinline__
#define CP_HDN inline __host__ __device__
#else
#define CP_HD inline
#define CP_HDN inline
#endif

namespace cp {
namespace pose {

struct PnPOut {
  int status;   // cp_pnp_status
  int n_pts;
  double loc[3];
  double quat[4];     // xyzw
  double reproj;
  double proj[16];    // 8 x (u, v) projected cuboid, OpenCV pose
  double kps3d[27];   // 9 x 3: centroid + 8 vertices in the returned frame
  double kpspnp[18];  // 9 x 2: (mean, 8 projected) / (width, height)
};

// ---- small dense helpers -------------------------------------------------------
CP_HD void mat3_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
}

CP_HD double mat3_det(const double* A) {
  return A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
}

// inverse-transpose of a 3x3 (cofactor matrix / det)
CP_HD void mat3_inv_t(const double* A, double* Bt) {
  double d = mat3_det(A);
  double id = 1.0 / d;
  Bt[0] = (A[4] * A[8] - A[5] * A[7]) * id;
  Bt[1] = (A[5] * A[6] - A[3] * A[8]) * id;
  Bt[2] = (A[3] * A[7] - A[4] * A[6]) * id;
  Bt[3] = (A[2] * A[7] - A[1] * A[8]) * id;
  Bt[4] = (A[0] * A[8] - A[2] * A[6]) * id;
  Bt[5] = (A[1] * A[6] - A[0] * A[7]) * id;
  Bt[6] = (A[1] * A[5] - A[2] * A[4]) * id;
  Bt[7] = (A[2] * A[3] - A[0] * A[5]) * id;
  Bt[8] = (A[0] * A[4] - A[1] * A[3]) * id;
}

// exp([w]x) -- Rodrigues
CP_HD void rodrigues(const double* w, double* R) {
  double th = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  if (th < 1e-300) {
    for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    return;
  }
  const double ith = 1.0 / th;
  double kx = w[0] * ith, ky = w[1] * ith, kz = w[2] * ith;
  double s = sin(th), c1 = 1.0 - cos(th);
  double K[9] = {0, -kz, ky, kz, 0, -kx, -ky, kx, 0};
  double K2[9];
  mat3_mul(K, K, K2);
  for (int i = 0; i < 9; ++i) R[i] = ((i % 4 == 0) ? 1.0 : 0.0) + s * K[i] + c1 * K2[i];
}

// rotation matrix -> unit quaternion xyzw with w >= 0
CP_HD void mat_to_quat(const double* R, double* q) {
  double tr = R[0] + R[4] + R[8];
  double c[4] = {R[0], R[4], R[8], tr};
  int i = 0;
  for (int t = 1; t < 4; ++t)
    if (c[t] > c[i]) i = t;
  if (i == 3) {
    q[3] = 1 + tr;
    q[0] = R[7] - R[5];
    q[1] = R[2] - R[6];
    q[2] = R[3] - R[1];
  } else {
    int j = (i + 1) % 3, k = (i + 2) % 3;
    q[i] = 1 - tr + 2 * R[i * 3 + i];
    q[j] = R[j * 3 + i] + R[i * 3 + j];
    q[k] = R[k * 3 + i] + R[i * 3 + k];
    q[3] = R[k * 3 + j] - R[j * 3 + k];
  }
  double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  double s = (q[3] < 0 ? -1.0 : 1.0) / n;
  for (int t = 0; t < 4; ++t) q[t] *= s;
}

CP_HD void quat_to_mat(const double* q, double* R) {
  double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
  R[0] = 1 - 2 * (y * y + z * z);
  R[1] = 2 * (x * y - z * w);
  R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w);
  R[4] = 1 - 2 * (x * x + z * z);
  R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w);
  R[7] = 2 * (y * z + x * w);
  R[8] = 1 - 2 * (x * x + y * y);
}

// Cuboid3d(scale / scale[1]).get_vertices() -- float32 arithmetic, then widened
CP_HD void cuboid_vertices(const float* scale, double* V /*[8][3]*/) {
  float sy = scale[1];
  float w = (1.0f * scale[0]) / sy, h = (1.0f * scale[1]) / sy, d = (1.0f * scale[2]) / sy;
  float hx = w / 2.0f, hy = h / 2.0f, hz = d / 2.0f;
  int t = 0;
  for (int ix = 0; ix < 2; ++ix)
    for (int iy = 0; iy < 2; ++iy)
      for (int iz = 0; iz < 2; ++iz) {
        V[t * 3 + 0] = (double)(ix ? hx : -hx);
        V[t * 3 + 1] = (double)(iy ? hy : -hy);
        V[t * 3 + 2] = (double)(iz ? hz : -hz);
        ++t;
      }
}

// cyclic Jacobi eigen-decomposition of a symmetric N x N matrix (row-major, destroyed: eigenvalues end on the diagonal);
// the eigenvectors are the COLUMNS of V.
template <int N>
CP_HDN void jacobi_eig(double* A, double* V) {
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) V[i * N + j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 60; ++sweep) {
    double off = 0.0, diag = 0.0;
    for (int i = 0; i < N; ++i) {
      diag += A[i * N + i] * A[i * N + i];
      for (int j = i + 1; j < N; ++j) off += A[i * N + j] * A[i * N + j];
    }
    if (off <= 1e-60 * diag || off == 0.0) break;
    for (int p = 0; p < N - 1; ++p)
      for (int q = p + 1; q < N; ++q) {
        double apq = A[p * N + q];
        if (apq == 0.0) continue;
        double app = A[p * N + p], aqq = A[q * N + q];
        double theta = (aqq - app) / (2.0 * apq);
        double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < N; ++k) {
          double akp = A[k * N + p], akq = A[k * N + q];
          A[k * N + p] = c * akp - s * akq;
          A[k * N + q] = s * akp + c * akq;
        }
        for (int k = 0; k < N; ++k) {
          double apk = A[p * N + k], aqk = A[q * N + k];
          A[p * N + k] = c * apk - s * aqk;
          A[q * N + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < N; ++k) {
          double vkp = V[k * N + p], vkq = V[k * N + q];
          V[k * N + p] = c * vkp - s * vkq;
          V[k * N + q] = s * vkp + c * vkq;
        }
      }
  }
}

// returns the eigenvector of the smallest eigenvalue in `vmin`.
template <int N>
CP_HDN void jacobi_min_eigvec(double* A, double* V, double* vmin) {
  jacobi_eig<N>(A, V);
  int m = 0;
  for (int i = 1; i < N; ++i)
    if (A[i * N + i] < A[m * N + m]) m = i;
  for (int k = 0; k < N; ++k) vmin[k] = V[k * N + m];
}

// solve the symmetric positive-definite 6x6 system (A + lam*diag(A)) d = -g by Cholesky; false if not SPD
CP_HDN bool solve6(const double* A, const double* g, double lam, double* d) {
  // one reciprocal per pivot instead of a division per entry: on the GPU an fp64 division is a ~20-instruction dependent
  // sequence and this routine sits inside the LM loop of every object (27 divisions -> 6)
  double L[36], inv[6];
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j <= i; ++j) {
      double s = A[i * 6 + j];
      if (i == j) s += lam * A[i * 6 + i];
      for (int k = 0; k < j; ++k) s -= L[i * 6 + k] * L[j * 6 + k];
      if (i == j) {
        if (!(s > 0.0)) return false;
        L[i * 6 + i] = sqrt(s);
        inv[i] = 1.0 / L[i * 6 + i];
      } else {
        L[i * 6 + j] = s * inv[j];
      }
    }
  double y[6];
  for (int i = 0; i < 6; ++i) {
    double s = -g[i];
    for (int k = 0; k < i; ++k) s -= L[i * 6 + k] * y[k];
    y[i] = s * inv[i];
  }
  for (int i = 5; i >= 0; --i) {
    double s = y[i];
    for (int k = i + 1; k < 6; ++k) s -= L[k * 6 + i] * d[k];
    d[i] = s * inv[i];
  }
  return true;
}

CP_HD double reproj_cost(const double* X, const double* uv, int n, const double* R, const double* t, double fx,
                         double fy, double cx, double cy) {
  double c = 0.0;
  for (int i = 0; i < n; ++i) {
    const double* x = X + 3 * i;
    double px = R[0] * x[0] + R[1] * x[1] + R[2] * x[2] + t[0];
    double py = R[3] * x[0] + R[4] * x[1] + R[5] * x[2] + t[1];
    double pz = R[6] * x[0] + R[7] * x[1] + R[8] * x[2] + t[2];
    double du = fx * px / pz + cx - uv[2 * i];
    double dv = fy * py / pz + cy - uv[2 * i + 1];
    c += du * du + dv * dv;
  }
  return c;
}

// second half of the DLT start: null vector p (3x4 projection, row-major) -> nearest rotation + scaled translation
CP_HDN void dlt_finish(const double* p, double* R, double* t) {
  double RR[9] = {p[0], p[1], p[2], p[4], p[5], p[6], p[8], p[9], p[10]};
  double tt[3] = {p[3], p[7], p[11]};
  if (mat3_det(RR) < 0) {
    for (int i = 0; i < 9; ++i) RR[i] = -RR[i];
    for (int i = 0; i < 3; ++i) tt[i] = -tt[i];
  }
  double sc = 0.0;
  for (int i = 0; i < 9; ++i) sc += RR[i] * RR[i];
  sc = sqrt(sc);
  // orthogonal polar factor U V^T of RR by Newton iteration X <- (X + X^-T) / 2
  double Xm[9];
  for (int i = 0; i < 9; ++i) Xm[i] = RR[i] / sc * 1.7320508075688772;
  for (int it = 0; it < 40; ++it) {
    double Xit[9];
    mat3_inv_t(Xm, Xit);
    double diff = 0.0;
    for (int i = 0; i < 9; ++i) {
      double nx = 0.5 * (Xm[i] + Xit[i]);
      diff += (nx - Xm[i]) * (nx - Xm[i]);
      Xm[i] = nx;
    }
    if (diff < 1e-30) break;
  }
  for (int i = 0; i < 9; ++i) R[i] = Xm[i];
  double f = 1.7320508075688772 / sc;  // ||R_orth||_F / ||RR||_F
  for (int i = 0; i < 3; ++i) t[i] = tt[i] * f;
}

// DLT start (OpenCV findExtrinsicCameraParams2, non-planar branch)
CP_HDN void dlt_init(const double* X, const double* uv, int n, double fx, double fy, double cx, double cy, double* R,
                     double* t) {
  double A[144];
  for (int i = 0; i < 144; ++i) A[i] = 0.0;
  for (int i = 0; i < n; ++i) {
    double x = (uv[2 * i] - cx) / fx, y = (uv[2 * i + 1] - cy) / fy;
    double Xi = X[3 * i], Yi = X[3 * i + 1], Zi = X[3 * i + 2];
    double r1[12] = {Xi, Yi, Zi, 1, 0, 0, 0, 0, -x * Xi, -x * Yi, -x * Zi, -x};
    double r2[12] = {0, 0, 0, 0, Xi, Yi, Zi, 1, -y * Xi, -y * Yi, -y * Zi, -y};
    for (int a = 0; a < 12; ++a)
      for (int b = 0; b < 12; ++b) A[a * 12 + b] += r1[a] * r1[b] + r2[a] * r2[b];
  }
  double V[144], p[12];
  jacobi_min_eigvec<12>(A, V, p);
  dlt_finish(p, R, t);
}

// Levenberg-Marquardt on the pixel reprojection error, update R <- exp([dw]x) R, t <- t + dt
CP_HDN double refine_lm(const double* X, const double* uv, int n, double fx, double fy, double cx, double cy, double* R,
                        double* t) {
  double lam = 1e-3;
  double cost = reproj_cost(X, uv, n, R, t, fx, fy, cx, cy);
  // cv2's SOLVEPNP_ITERATIVE runs its LM under TermCriteria(MAX_ITER + EPS, 20, FLT_EPSILON).  Well-posed inputs
  // converge in < 10 steps (agreement with cv2 <= 5e-8); on inconsistent keypoints cv2 stops unconverged, and stopping
  // after 20 accepted steps stays closest to what it returns (measured: |dR| 2e-2 vs 6e-1 for a 200-step run).
  for (int iter = 0; iter < 20; ++iter) {
    double A[36], g[6];
    for (int i = 0; i < 36; ++i) A[i] = 0.0;
    for (int i = 0; i < 6; ++i) g[i] = 0.0;
    for (int i = 0; i < n; ++i) {
      const double* x = X + 3 * i;
      double qx = R[0] * x[0] + R[1] * x[1] + R[2] * x[2];
      double qy = R[3] * x[0] + R[4] * x[1] + R[5] * x[2];
      double qz = R[6] * x[0] + R[7] * x[1] + R[8] * x[2];
      double px = qx + t[0], py = qy + t[1], pz = qz + t[2];
      double iz = 1.0 / pz;
      double du[3] = {fx * iz, 0.0, -fx * px * iz * iz};
      double dv[3] = {0.0, fy * iz, -fy * py * iz * iz};
      // dP/dw = -[q]x  ->  row . (-[q]x) = (q x row)^T ... written out:
      double Ju[6], Jv[6];
      // -[q]x = [[0, qz, -qy], [-qz, 0, qx], [qy, -qx, 0]]
      Ju[0] = du[1] * (-qz) + du[2] * qy;
      Ju[1] = du[0] * qz + du[2] * (-qx);
      Ju[2] = du[0] * (-qy) + du[1] * qx;
      Jv[0] = dv[1] * (-qz) + dv[2] * qy;
      Jv[1] = dv[0] * qz + dv[2] * (-qx);
      Jv[2] = dv[0] * (-qy) + dv[1] * qx;
      for (int k = 0; k < 3; ++k) {
        Ju[3 + k] = du[k];
        Jv[3 + k] = dv[k];
      }
      double ru = fx * px * iz + cx - uv[2 * i];
      double rv = fy * py * iz + cy - uv[2 * i + 1];
      for (int a = 0; a < 6; ++a) {
        g[a] += Ju[a] * ru + Jv[a] * rv;
        for (int b = 0; b <= a; ++b) A[a * 6 + b] += Ju[a] * Ju[b] + Jv[a] * Jv[b];
      }
    }
    for (int a = 0; a < 6; ++a)
      for (int b = a + 1; b < 6; ++b) A[a * 6 + b] = A[b * 6 + a];
    bool improved = false;
    double d[6], Rn[9], tn[3], cn = 0.0;
    for (int tr = 0; tr < 30; ++tr) {
      if (solve6(A, g, lam, d)) {
        double E[9];
        rodrigues(d, E);
        mat3_mul(E, R, Rn);
        for (int k = 0; k < 3; ++k) tn[k] = t[k] + d[3 + k];
        cn = reproj_cost(X, uv, n, Rn, tn, fx, fy, cx, cy);
        if (cn == cn && cn <= cost && fabs(cn) < 1e300) {
          improved = true;
          break;
        }
      }
      lam *= 10.0;
    }
    if (!improved) break;
    double step = 0.0;
    for (int k = 0; k < 6; ++k) step += d[k] * d[k];
    step = sqrt(step);
    for (int k = 0; k < 9; ++k) R[k] = Rn[k];
    for (int k = 0; k < 3; ++k) t[k] = tn[k];
    double dec = cost - cn;
    cost = cn;
    lam = lam * 0.1;
    if (lam < 1e-12) lam = 1e-12;
    if (step < 1e-10 || dec <= 1e-28 * (cost > 1e-300 ? cost : 1e-300)) break;
  }
  return cost;
}


// ---- EPnP (Lepetit, Moreno-Noguer, Fua, IJCV 2009) for 4 - 5 valid points -------------------------------------------------
// cuboid_pnp_solver.py:157-171 switches to cv2.SOLVEPNP_EPNP below 6 points (third party: OpenCV calib3d epnp.cpp, whose
// published algorithm is restated here: 4 control points from the PCA of the object points, barycentric coordinates,
// the 2n x 12 system M, its 4 smallest right singular vectors, the three beta approximations, 5 Gauss-Newton steps each,
// absolute orientation, best reprojection error).  With 4 or 5 points M has rank <= 2n < 12: the null space is 4- / 2-
// dimensional BY CONSTRUCTION and any orthonormal basis of it is a valid set of "smallest singular vectors" -- OpenCV
// takes whatever LAPACK returns, this code what the Jacobi sweep returns.  The two agree to 1e-12 on consistent 5-point
// input; on 4 points and on noisy input both return a valid EPnP pose but not the same one (tests/test_pose_core_host.py
// pins the consistent case against cv2 and bounds the reprojection error otherwise).
CP_HDN bool lstsq_small(const double* A, const double* b, int m, int n, double* x) {      // min |A x - b|, n <= 5, via normal equations + pivoted elimination
  double N[25], g[5];
  for (int i = 0; i < n; ++i) {
    g[i] = 0.0;
    for (int r = 0; r < m; ++r) g[i] += A[r * n + i] * b[r];
    for (int j = 0; j < n; ++j) {
      double s = 0.0;
      for (int r = 0; r < m; ++r) s += A[r * n + i] * A[r * n + j];
      N[i * n + j] = s;
    }
  }
  // Tikhonov floor keeps the rank-deficient approximations of the 4 / 5 point case finite (pinv-like behaviour)
  double tr = 0.0;
  for (int i = 0; i < n; ++i) tr += N[i * n + i];
  for (int i = 0; i < n; ++i) N[i * n + i] += 1e-13 * tr + 1e-300;
  for (int c = 0; c < n; ++c) {
    int piv = c;
    for (int r = c + 1; r < n; ++r)
      if (fabs(N[r * n + c]) > fabs(N[piv * n + c])) piv = r;
    if (N[piv * n + c] == 0.0) return false;
    if (piv != c) {
      for (int j = 0; j < n; ++j) {
        const double t = N[c * n + j];
        N[c * n + j] = N[piv * n + j];
        N[piv * n + j] = t;
      }
      const double t = g[c];
      g[c] = g[piv];
      g[piv] = t;
    }
    for (int r = c + 1; r < n; ++r) {
      const double f = N[r * n + c] / N[c * n + c];
      for (int j = c; j < n; ++j) N[r * n + j] -= f * N[c * n + j];
      g[r] -= f * g[c];
    }
  }
  for (int i = n - 1; i >= 0; --i) {
    double s = g[i];
    for (int j = i + 1; j < n; ++j) s -= N[i * n + j] * x[j];
    x[i] = s / N[i * n + i];
  }
  return true;
}

CP_HD double dot3(const double* p, const double* q) { return p[0] * q[0] + p[1] * q[1] + p[2] * q[2]; }

// absolute orientation of the camera-frame points pcs against the object points X (epnp.cpp estimate_R_and_t):
// R = U V^T of sum (pc - pc0)(pw - pw0)^T through the polar factor, det fixed by flipping the last row
CP_HDN void epnp_rt(const double* X, const double* pcs, int n, double* R, double* t) {
  double pc0[3] = {0, 0, 0}, pw0[3] = {0, 0, 0};
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < 3; ++k) {
      pc0[k] += pcs[3 * i + k] / n;
      pw0[k] += X[3 * i + k] / n;
    }
  double H[9];
  for (int i = 0; i < 9; ++i) H[i] = 0.0;
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < 3; ++j)
      for (int k = 0; k < 3; ++k) H[j * 3 + k] += (pcs[3 * i + j] - pc0[j]) * (X[3 * i + k] - pw0[k]);
  // U V^T = H (H^T H)^(-1/2): eigen-decomposition of the symmetric 3 x 3 H^T H
  double S[9], E[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) S[i * 3 + j] = H[0 * 3 + i] * H[0 * 3 + j] + H[1 * 3 + i] * H[1 * 3 + j] + H[2 * 3 + i] * H[2 * 3 + j];
  jacobi_eig<3>(S, E);
  // order the eigenvalues descending; a (near-)zero smallest one (coplanar points) is completed by the cross product
  int o[3] = {0, 1, 2};
  for (int a = 0; a < 2; ++a)
    for (int b = a + 1; b < 3; ++b)
      if (S[o[b] * 3 + o[b]] > S[o[a] * 3 + o[a]]) {
        const int tt = o[a];
        o[a] = o[b];
        o[b] = tt;
      }
  double Vc[3][3], Uc[3][3];      // columns
  for (int c = 0; c < 3; ++c)
    for (int k = 0; k < 3; ++k) Vc[c][k] = E[k * 3 + o[c]];
  const double big = S[o[0] * 3 + o[0]];
  for (int c = 0; c < 2; ++c) {
    const double sv = sqrt(fmax(S[o[c] * 3 + o[c]], 0.0));
    for (int k = 0; k < 3; ++k) Uc[c][k] = (H[k * 3] * Vc[c][0] + H[k * 3 + 1] * Vc[c][1] + H[k * 3 + 2] * Vc[c][2]) / (sv > 0 ? sv : 1.0);
  }
  const double s2 = sqrt(fmax(S[o[2] * 3 + o[2]], 0.0));
  if (s2 > 1e-9 * sqrt(fmax(big, 1e-300))) {
    for (int k = 0; k < 3; ++k) Uc[2][k] = (H[k * 3] * Vc[2][0] + H[k * 3 + 1] * Vc[2][1] + H[k * 3 + 2] * Vc[2][2]) / s2;
  } else {
    Uc[2][0] = Uc[0][1] * Uc[1][2] - Uc[0][2] * Uc[1][1];
    Uc[2][1] = Uc[0][2] * Uc[1][0] - Uc[0][0] * Uc[1][2];
    Uc[2][2] = Uc[0][0] * Uc[1][1] - Uc[0][1] * Uc[1][0];
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) R[i * 3 + j] = Uc[0][i] * Vc[0][j] + Uc[1][i] * Vc[1][j] + Uc[2][i] * Vc[2][j];
  if (mat3_det(R) < 0) {
    R[6] = -R[6];
    R[7] = -R[7];
    R[8] = -R[8];
  }
  for (int k = 0; k < 3; ++k) t[k] = pc0[k] - (R[k * 3] * pw0[0] + R[k * 3 + 1] * pw0[1] + R[k * 3 + 2] * pw0[2]);
}

// EPnP in three steps, so that the CUDA kernels can run the 12 x 12 eigen-decomposition warp-cooperatively (pnp_warp.cuh)
// while the host runs the serial chain epnp_solve below:
//   epnp_prepare    control points (centroid + principal directions) and barycentric coordinates of the object points
//   epnp_mtm_entry  one entry of M^T M (12 x 12), accumulated over the points in order
//   epnp_finish     from the eigen-decomposition of M^T M to the pose (betas, Gauss-Newton, absolute orientation)
struct EpnpPre {
  double cws[4][3];
  double al[16][4];
};

CP_HDN bool epnp_prepare(const double* X, int n, EpnpPre* P) {
  // control points: centroid + principal directions scaled by sqrt(eigenvalue / n)
  double (*cws)[3] = P->cws;
  double (*al)[4] = P->al;
  for (int k = 0; k < 3; ++k) {
    cws[0][k] = 0.0;
    for (int i = 0; i < n; ++i) cws[0][k] += X[3 * i + k] / n;
  }
  double C[9], E[9];
  for (int i = 0; i < 9; ++i) C[i] = 0.0;
  for (int i = 0; i < n; ++i)
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) C[a * 3 + b] += (X[3 * i + a] - cws[0][a]) * (X[3 * i + b] - cws[0][b]);
  jacobi_eig<3>(C, E);
  int o[3] = {0, 1, 2};
  for (int a = 0; a < 2; ++a)
    for (int b = a + 1; b < 3; ++b)
      if (C[o[b] * 3 + o[b]] > C[o[a] * 3 + o[a]]) {
        const int tt = o[a];
        o[a] = o[b];
        o[b] = tt;
      }
  for (int i = 1; i < 4; ++i) {
    const double k = sqrt(fmax(C[o[i - 1] * 3 + o[i - 1]], 0.0) / n);
    for (int j = 0; j < 3; ++j) cws[i][j] = cws[0][j] + k * E[j * 3 + o[i - 1]];
  }
  // barycentric coordinates
  double CC[9], CCit[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 1; j < 4; ++j) CC[3 * i + j - 1] = cws[j][i] - cws[0][i];
  if (fabs(mat3_det(CC)) < 1e-300) return false;      // coplanar object points: EPnP's general case does not apply
  mat3_inv_t(CC, CCit);                               // CCit = (CC^-1)^T
  for (int i = 0; i < n; ++i) {
    const double d[3] = {X[3 * i] - cws[0][0], X[3 * i + 1] - cws[0][1], X[3 * i + 2] - cws[0][2]};
    for (int j = 0; j < 3; ++j) al[i][1 + j] = CCit[0 * 3 + j] * d[0] + CCit[1 * 3 + j] * d[1] + CCit[2 * 3 + j] * d[2];
    al[i][0] = 1.0 - al[i][1] - al[i][2] - al[i][3];
  }
  return true;
}

// entry (a, b) of M^T M: rows r1 = [al_j fx, 0, al_j (cx - u)], r2 = [0, al_j fy, al_j (cy - v)] (j = 0..3) per point
CP_HDN double epnp_mtm_entry(const EpnpPre& P, const double* uv, int n, double fx, double fy, double cx, double cy, int a,
                             int b) {
  const int ja = a / 3, ka = a - 3 * ja, jb = b / 3, kb = b - 3 * jb;
  double acc = 0.0;
  for (int i = 0; i < n; ++i) {
    const double du = cx - uv[2 * i], dv = cy - uv[2 * i + 1];
    const double r1a = ka == 0 ? P.al[i][ja] * fx : (ka == 1 ? 0.0 : P.al[i][ja] * du);
    const double r1b = kb == 0 ? P.al[i][jb] * fx : (kb == 1 ? 0.0 : P.al[i][jb] * du);
    const double r2a = ka == 0 ? 0.0 : (ka == 1 ? P.al[i][ja] * fy : P.al[i][ja] * dv);
    const double r2b = kb == 0 ? 0.0 : (kb == 1 ? P.al[i][jb] * fy : P.al[i][jb] * dv);
    acc += r1a * r1b + r2a * r2b;
  }
  return acc;
}

// MtM: the 12 x 12 matrix after its Jacobi eigen-decomposition (eigenvalues on the diagonal), V: eigenvectors in columns.
// Returns the mean reprojection error (pixels) of the chosen pose.
CP_HDN double epnp_finish(const double* X, const double* uv, int n, double fx, double fy, double cx, double cy,
                          const EpnpPre& P, const double* MtM, const double* V, double* Rout, double* tout) {
  const double (*cws)[3] = P.cws;
  const double (*al)[4] = P.al;
  int ord[12];
  for (int i = 0; i < 12; ++i) ord[i] = i;
  for (int a = 0; a < 4; ++a)                    // the four smallest eigenvalues, ascending
    for (int b = a + 1; b < 12; ++b)
      if (MtM[ord[b] * 12 + ord[b]] < MtM[ord[a] * 12 + ord[a]]) {
        const int tt = ord[a];
        ord[a] = ord[b];
        ord[b] = tt;
      }
  double v[4][12];
  for (int i = 0; i < 4; ++i)
    for (int k = 0; k < 12; ++k) v[i][k] = V[k * 12 + ord[i]];
  // L (6 x 10) and rho
  double dv[4][6][3];
  for (int i = 0; i < 4; ++i) {
    int a = 0, b = 1;
    for (int j = 0; j < 6; ++j) {
      for (int k = 0; k < 3; ++k) dv[i][j][k] = v[i][3 * a + k] - v[i][3 * b + k];
      if (++b > 3) {
        ++a;
        b = a + 1;
      }
    }
  }
  double L[60], rho[6];
  for (int i = 0; i < 6; ++i) {
    double* r = L + 10 * i;
    r[0] = dot3(dv[0][i], dv[0][i]);
    r[1] = 2 * dot3(dv[0][i], dv[1][i]);
    r[2] = dot3(dv[1][i], dv[1][i]);
    r[3] = 2 * dot3(dv[0][i], dv[2][i]);
    r[4] = 2 * dot3(dv[1][i], dv[2][i]);
    r[5] = dot3(dv[2][i], dv[2][i]);
    r[6] = 2 * dot3(dv[0][i], dv[3][i]);
    r[7] = 2 * dot3(dv[1][i], dv[3][i]);
    r[8] = 2 * dot3(dv[2][i], dv[3][i]);
    r[9] = dot3(dv[3][i], dv[3][i]);
  }
  {
    const int pa[6] = {0, 0, 0, 1, 1, 2}, pb[6] = {1, 2, 3, 2, 3, 3};
    for (int i = 0; i < 6; ++i) {
      double d = 0.0;
      for (int k = 0; k < 3; ++k) d += (cws[pa[i]][k] - cws[pb[i]][k]) * (cws[pa[i]][k] - cws[pb[i]][k]);
      rho[i] = d;
    }
  }
  double best = 1e300;
  for (int ap = 0; ap < 3; ++ap) {
    double be[4] = {0, 0, 0, 0};
    if (ap == 0) {            // betas ~ [B11 B12 B13 B14]
      const int cols[4] = {0, 1, 3, 6};
      double A4[24], b4[4];
      for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 4; ++j) A4[i * 4 + j] = L[10 * i + cols[j]];
      if (!lstsq_small(A4, rho, 6, 4, b4)) continue;
      if (b4[0] < 0) {
        be[0] = sqrt(-b4[0]);
        for (int j = 1; j < 4; ++j) be[j] = -b4[j] / be[0];
      } else {
        be[0] = sqrt(b4[0]);
        for (int j = 1; j < 4; ++j) be[j] = b4[j] / be[0];
      }
    } else {                  // [B11 B12 B22] / [B11 B12 B22 B13 B23]
      const int nc = ap == 1 ? 3 : 5;
      double A5[30], b5[5];
      for (int i = 0; i < 6; ++i)
        for (int j = 0; j < nc; ++j) A5[i * nc + j] = L[10 * i + j];
      if (!lstsq_small(A5, rho, 6, nc, b5)) continue;
      if (b5[0] < 0) {
        be[0] = sqrt(-b5[0]);
        be[1] = b5[2] < 0 ? sqrt(-b5[2]) : 0.0;
      } else {
        be[0] = sqrt(b5[0]);
        be[1] = b5[2] > 0 ? sqrt(b5[2]) : 0.0;
      }
      if (b5[1] < 0) be[0] = -be[0];
      if (ap == 2) be[2] = b5[3] / be[0];
    }
    if (!(be[0] == be[0]) || be[0] == 0.0) continue;
    for (int it = 0; it < 5; ++it) {          // Gauss-Newton on the six control-point distances
      double A[24], b[6], dx[4];
      for (int i = 0; i < 6; ++i) {
        const double* r = L + 10 * i;
        A[i * 4 + 0] = 2 * r[0] * be[0] + r[1] * be[1] + r[3] * be[2] + r[6] * be[3];
        A[i * 4 + 1] = r[1] * be[0] + 2 * r[2] * be[1] + r[4] * be[2] + r[7] * be[3];
        A[i * 4 + 2] = r[3] * be[0] + r[4] * be[1] + 2 * r[5] * be[2] + r[8] * be[3];
        A[i * 4 + 3] = r[6] * be[0] + r[7] * be[1] + r[8] * be[2] + 2 * r[9] * be[3];
        b[i] = rho[i] - (r[0] * be[0] * be[0] + r[1] * be[0] * be[1] + r[2] * be[1] * be[1] + r[3] * be[0] * be[2] +
                         r[4] * be[1] * be[2] + r[5] * be[2] * be[2] + r[6] * be[0] * be[3] + r[7] * be[1] * be[3] +
                         r[8] * be[2] * be[3] + r[9] * be[3] * be[3]);
      }
      if (!lstsq_small(A, b, 6, 4, dx)) break;
      for (int j = 0; j < 4; ++j) be[j] += dx[j];
    }
    // control points in the camera frame, the points themselves, sign, absolute orientation
    double ccs[4][3], pcs[48];
    for (int j = 0; j < 4; ++j)
      for (int k = 0; k < 3; ++k) ccs[j][k] = be[0] * v[0][3 * j + k] + be[1] * v[1][3 * j + k] + be[2] * v[2][3 * j + k] + be[3] * v[3][3 * j + k];
    for (int i = 0; i < n; ++i)
      for (int k = 0; k < 3; ++k) pcs[3 * i + k] = al[i][0] * ccs[0][k] + al[i][1] * ccs[1][k] + al[i][2] * ccs[2][k] + al[i][3] * ccs[3][k];
    if (pcs[2] < 0.0)
      for (int i = 0; i < 3 * n; ++i) pcs[i] = -pcs[i];
    double R[9], t[3];
    epnp_rt(X, pcs, n, R, t);
    double err = 0.0;
    bool fin = true;
    for (int i = 0; i < n; ++i) {
      const double* x = X + 3 * i;
      const double px = R[0] * x[0] + R[1] * x[1] + R[2] * x[2] + t[0];
      const double py = R[3] * x[0] + R[4] * x[1] + R[5] * x[2] + t[1];
      const double pz = R[6] * x[0] + R[7] * x[1] + R[8] * x[2] + t[2];
      const double du = cx + fx * px / pz - uv[2 * i], dvv = cy + fy * py / pz - uv[2 * i + 1];
      err += sqrt(du * du + dvv * dvv) / n;
    }
    fin = err == err;
    if (fin && err < best) {
      best = err;
      for (int i = 0; i < 9; ++i) Rout[i] = R[i];
      for (int i = 0; i < 3; ++i) tout[i] = t[i];
    }
  }
  return best;
}

// X: n x 3 object points, uv: n x 2 pixels (4 <= n <= 16).  Returns the mean reprojection error (pixels) of the chosen pose.
CP_HDN double epnp_solve(const double* X, const double* uv, int n, double fx, double fy, double cx, double cy, double* Rout,
                         double* tout) {
  EpnpPre P;
  if (!epnp_prepare(X, n, &P)) return 1e300;
  double MtM[144], V[144];
  for (int a = 0; a < 12; ++a)
    for (int b = 0; b < 12; ++b) MtM[a * 12 + b] = epnp_mtm_entry(P, uv, n, fx, fy, cx, cy, a, b);
  jacobi_eig<12>(MtM, V);
  return epnp_finish(X, uv, n, fx, fy, cx, cy, P, MtM, V, Rout, tout);
}

// solve_pnp + pnp_shell for one detection, in three steps so that the CUDA decode kernel can run the two heavy ones
// (DLT eigen-solve, LM) warp-cooperatively (decode.cu) while host tests run the serial chain below.
//   pts: n_in x 2 image points (n_in = 8 or 16; 3-D vertex of point i is V[i / (n_in/8)])
//   Kc:  camera matrix row-major; width/height: image size for kps_pnp normalisation
//   visible_thresh: 6 / 3 / 0 (see cp_decode_params)
// pnp_collect: cuboid vertices + the points that are not the -10000 sentinel; returns their number.
// same with the vertices given (tracker: the pooled scale is float64, so are its vertices -- tracker.py:263-273)
CP_HDN int pnp_collect_v(const double* pts, int n_in, const double* V /*24*/, double* X /*48*/, double* uv /*32*/) {
  int n = 0;
  const int per = n_in / 8;
  for (int i = 0; i < n_in; ++i) {
    if (pts[2 * i] < -5000.0 || pts[2 * i + 1] < -5000.0) continue;
    uv[2 * n] = pts[2 * i];
    uv[2 * n + 1] = pts[2 * i + 1];
    const double* v = V + 3 * (i / per);
    X[3 * n] = v[0];
    X[3 * n + 1] = v[1];
    X[3 * n + 2] = v[2];
    ++n;
  }
  return n;
}

// Cuboid3d(scale / scale[1]).get_vertices() in float64 (scale is a float64 array there)
CP_HD void cuboid_vertices_d(const double* scale, double* V /*[8][3]*/) {
  const double hx = (scale[0] / scale[1]) / 2.0, hy = (scale[1] / scale[1]) / 2.0, hz = (scale[2] / scale[1]) / 2.0;
  int t = 0;
  for (int ix = 0; ix < 2; ++ix)
    for (int iy = 0; iy < 2; ++iy)
      for (int iz = 0; iz < 2; ++iz) {
        V[t * 3 + 0] = ix ? hx : -hx;
        V[t * 3 + 1] = iy ? hy : -hy;
        V[t * 3 + 2] = iz ? hz : -hz;
        ++t;
      }
}

CP_HDN int pnp_collect(const double* pts, int n_in, const float* obj_scale, double* V /*24*/, double* X /*48*/,
                       double* uv /*32*/) {
  cuboid_vertices(obj_scale, V);
  int n = 0;
  const int per = n_in / 8;
  for (int i = 0; i < n_in; ++i) {
    if (pts[2 * i] < -5000.0 || pts[2 * i + 1] < -5000.0) continue;
    uv[2 * n] = pts[2 * i];
    uv[2 * n + 1] = pts[2 * i + 1];
    const double* v = V + 3 * (i / per);
    X[3 * n] = v[0];
    X[3 * n + 1] = v[1];
    X[3 * n + 2] = v[2];
    ++n;
  }
  return n;
}

// The visibility gate of cuboid_pnp_shell.py:59-79: at least visible_thresh of the nine projected points (kps_pnp,
// normalised) outside the image makes a pose invisible; visible_thresh <= 0 turns the gate off.
CP_HD bool pnp_gate_invisible(const double* kpspnp, int visible_thresh) {
  if (visible_thresh <= 0) return false;
  int nv = 0;
  for (int i = 0; i < 9; ++i) {
    double a = kpspnp[2 * i], b = kpspnp[2 * i + 1];
    if (a < 0 || a > 1 || b < 0 || b > 1) ++nv;
  }
  return nv >= visible_thresh;
}

// pnp_finish: everything after the solver (cuboid_pnp_solver.py:190-239, cuboid_pnp_shell.py:24-93)
CP_HDN void pnp_finish(const double* V, const double* R, const double* t, double cost, int n, const double* Kc,
                       double width, double height, int visible_thresh, int opencv_return, PnPOut* o) {
  const double fx = Kc[0], fy = Kc[4], cx = Kc[2], cy = Kc[5];
  // a NaN or +-inf pose is a solver failure (pnp_ref.solve_pnp: np.isfinite); `fabs(x) <= DBL_MAX` is false for both
  bool finite = (cost == cost) && fabs(cost) < 1e300;
  for (int i = 0; i < 9; ++i) finite = finite && (fabs(R[i]) <= 1.7976931348623157e308);
  for (int i = 0; i < 3; ++i) finite = finite && (fabs(t[i]) <= 1.7976931348623157e308);
  if (!finite) {
    o->status = 5;
    return;
  }
  o->reproj = sqrt(cost / (2.0 * n));
  for (int i = 0; i < 8; ++i) {
    const double* x = V + 3 * i;
    double px = R[0] * x[0] + R[1] * x[1] + R[2] * x[2] + t[0];
    double py = R[3] * x[0] + R[4] * x[1] + R[5] * x[2] + t[1];
    double pz = R[6] * x[0] + R[7] * x[1] + R[8] * x[2] + t[2];
    o->proj[2 * i] = fx * px / pz + cx;
    o->proj[2 * i + 1] = fy * py / pz + cy;
  }
  if (t[2] < 0.0) {
    o->status = 3;  // CP_PNP_BEHIND
    return;
  }
  double Rr[9], tr[3];
  if (opencv_return) {
    for (int i = 0; i < 9; ++i) Rr[i] = R[i];
    for (int i = 0; i < 3; ++i) tr[i] = t[i];
  } else {
    // M = [[0,1,0],[1,0,0],[0,0,-1]]
    for (int j = 0; j < 3; ++j) {
      Rr[j] = R[3 + j];
      Rr[3 + j] = R[j];
      Rr[6 + j] = -R[6 + j];
    }
    tr[0] = t[1];
    tr[1] = t[0];
    tr[2] = -t[2];
  }
  mat_to_quat(Rr, o->quat);
  for (int i = 0; i < 3; ++i) o->loc[i] = tr[i];
  // kps_3d_cam = [mean, R(q) V + loc]
  double Rq[9];
  quat_to_mat(o->quat, Rq);
  double m3[3] = {0, 0, 0};
  for (int i = 0; i < 8; ++i) {
    const double* x = V + 3 * i;
    for (int k = 0; k < 3; ++k) {
      double v = Rq[k * 3] * x[0] + Rq[k * 3 + 1] * x[1] + Rq[k * 3 + 2] * x[2] + tr[k];
      o->kps3d[3 * (i + 1) + k] = v;
      m3[k] += v;
    }
  }
  for (int k = 0; k < 3; ++k) o->kps3d[k] = m3[k] / 8.0;
  double mu = 0, mv = 0;
  for (int i = 0; i < 8; ++i) {
    mu += o->proj[2 * i];
    mv += o->proj[2 * i + 1];
  }
  o->kpspnp[0] = (mu / 8.0) / width;
  o->kpspnp[1] = (mv / 8.0) / height;
  for (int i = 0; i < 8; ++i) {
    o->kpspnp[2 * (i + 1)] = o->proj[2 * i] / width;
    o->kpspnp[2 * (i + 1) + 1] = o->proj[2 * i + 1] / height;
  }
  o->status = 1;
  if (pnp_gate_invisible(o->kpspnp, visible_thresh)) o->status = 2;
  if (!(o->kpspnp[0] > 0 && o->kpspnp[0] < 1 && o->kpspnp[1] > 0 && o->kpspnp[1] < 1)) o->status = 2;
}

// 4 - 5 valid points: cv2.SOLVEPNP_EPNP (cuboid_pnp_solver.py:162-163), no iterative refinement
CP_HDN void pnp_few_points(const double* V, const double* X, const double* uv, int n, const double* Kc, double width,
                           double height, int visible_thresh, int opencv_return, PnPOut* o) {
  double R[9], t[3];
  const double err = epnp_solve(X, uv, n, Kc[0], Kc[4], Kc[2], Kc[5], R, t);
  if (!(err < 1e299)) {
    o->status = 5;  // CP_PNP_SOLVER_FAIL
    return;
  }
  pnp_finish(V, R, t, reproj_cost(X, uv, n, R, t, Kc[0], Kc[4], Kc[2], Kc[5]), n, Kc, width, height, visible_thresh,
             opencv_return, o);
}

CP_HDN void solve_and_shell(const double* pts, int n_in, const float* obj_scale, const double* Kc, double width,
                            double height, int visible_thresh, int opencv_return, PnPOut* o) {
  double V[24], X[48], uv[32];
  const int n = pnp_collect(pts, n_in, obj_scale, V, X, uv);
  o->n_pts = n;
  o->status = 4;  // CP_PNP_FEW_POINTS
  if (n < 4) return;
  if (n < 6) {
    pnp_few_points(V, X, uv, n, Kc, width, height, visible_thresh, opencv_return, o);
    return;
  }
  double R[9], t[3];
  dlt_init(X, uv, n, Kc[0], Kc[4], Kc[2], Kc[5], R, t);
  const double cost = refine_lm(X, uv, n, Kc[0], Kc[4], Kc[2], Kc[5], R, t);
  pnp_finish(V, R, t, cost, n, Kc, width, height, visible_thresh, opencv_return, o);
}

// solve_and_shell with the cuboid vertices given
CP_HDN void solve_and_shell_v(const double* pts, int n_in, const double* V, const double* Kc, double width, double height,
                              int visible_thresh, int opencv_return, PnPOut* o) {
  double X[48], uv[32];
  const int n = pnp_collect_v(pts, n_in, V, X, uv);
  o->n_pts = n;
  o->status = 4;  // CP_PNP_FEW_POINTS
  if (n < 4) return;
  if (n < 6) {
    pnp_few_points(V, X, uv, n, Kc, width, height, visible_thresh, opencv_return, o);
    return;
  }
  double R[9], t[3];
  dlt_init(X, uv, n, Kc[0], Kc[4], Kc[2], Kc[5], R, t);
  const double cost = refine_lm(X, uv, n, Kc[0], Kc[4], Kc[2], Kc[5], R, t);
  pnp_finish(V, R, t, cost, n, Kc, width, height, visible_thresh, opencv_return, o);
}

// ---- Gaussian soft-NMS (object_pose.py:27-124, method=2, sigma=0.5) ----------------
// bbox: n x 4 doubles, score: n doubles, perm: n ints (identity on entry).  On exit the
// first return-value entries of perm/score are the survivors in the reference's order.
CP_HDN int soft_nms(double* bbox, double* score, int* perm, int n, double threshold) {
  int N = n;
  for (int i = 0; i < N; ++i) {
    int maxpos = i;
    double maxscore = score[i];
    for (int pos = i + 1; pos < N; ++pos)
      if (maxscore < score[pos]) {
        maxscore = score[pos];
        maxpos = pos;
      }
    if (maxpos != i) {
      for (int k = 0; k < 4; ++k) {
        double tmp = bbox[4 * i + k];
        bbox[4 * i + k] = bbox[4 * maxpos + k];
        bbox[4 * maxpos + k] = tmp;
      }
      double ts = score[i];
      score[i] = score[maxpos];
      score[maxpos] = ts;
      int tp = perm[i];
      perm[i] = perm[maxpos];
      perm[maxpos] = tp;
    }
    double tx1 = bbox[4 * i], ty1 = bbox[4 * i + 1], tx2 = bbox[4 * i + 2], ty2 = bbox[4 * i + 3];
    int pos = i + 1;
    while (pos < N) {
      double x1 = bbox[4 * pos], y1 = bbox[4 * pos + 1], x2 = bbox[4 * pos + 2], y2 = bbox[4 * pos + 3];
      double area = (x2 - x1 + 1) * (y2 - y1 + 1);
      double iw = fmin(tx2, x2) - fmax(tx1, x1) + 1;
      if (iw > 0) {
        double ih = fmin(ty2, y2) - fmax(ty1, y1) + 1;
        if (ih > 0) {
          double ua = (tx2 - tx1 + 1) * (ty2 - ty1 + 1) + area - iw * ih;
          double ov = iw * ih / ua;
          double weight = exp(-(ov * ov) / 0.5);
          score[pos] = weight * score[pos];
          if (score[pos] < threshold) {
            for (int k = 0; k < 4; ++k) bbox[4 * pos + k] = bbox[4 * (N - 1) + k];
            score[pos] = score[N - 1];
            int tp = perm[pos];
            perm[pos] = perm[N - 1];
            perm[N - 1] = tp;
            N -= 1;
            pos -= 1;
          }
        }
      }
      pos += 1;
    }
  }
  return N;
}

// ---- gpfit.moments on a (nr x nc) window of doubles (row-major, ld = nc) ----------------
// returns false when the reference would raise: an empty window, a NaN centroid, a centroid row / column index outside
// the window, or a start point that fitgaussian's least_squares(bounds=(0, [inf, nr, nc, inf, inf])) rejects as
// infeasible (a negative height, a centroid outside [0, nr] x [0, nc], a NaN or negative width).  Raw (opt.mse_loss)
// windows with a non-positive total or a non-positive centroid row / column sum end here.
CP_HDN bool moments(const double* w, int nr, int nc, double* height, double* x, double* y, double* wx, double* wy) {
  if (nr <= 0 || nc <= 0) return false;
  double total = 0, sx = 0, sy = 0, mx = w[0];
  for (int r = 0; r < nr; ++r)
    for (int c = 0; c < nc; ++c) {
      double v = w[r * nc + c];
      total += v;
      sx += r * v;
      sy += c * v;
      if (v > mx) mx = v;
    }
  double xc = sx / total, yc = sy / total;
  if (!(xc == xc) || !(yc == yc)) return false;
  int iy = (int)yc, ix = (int)xc;  // truncation toward zero like int()
  if (iy < 0) iy += nc;            // python negative index
  if (ix < 0) ix += nr;
  if (iy < 0 || iy >= nc || ix < 0 || ix >= nr) return false;
  double num = 0, den = 0;
  for (int r = 0; r < nr; ++r) {
    double v = w[r * nc + iy];
    num += fabs((r - yc) * (r - yc) * v);
    den += v;
  }
  const double wxv = sqrt(num / den);  // np.abs(...).sum(): abs per term (raw windows mix signs), then the sum
  num = 0;
  den = 0;
  for (int c = 0; c < nc; ++c) {
    double v = w[ix * nc + c];
    num += fabs((c - xc) * (c - xc) * v);
    den += v;
  }
  const double wyv = sqrt(num / den);
  // the bounds test of least_squares, in_bounds(x0, lb, ub); every comparison with NaN is false
  if (!(mx >= 0.0 && xc >= 0.0 && xc <= (double)nr && yc >= 0.0 && yc <= (double)nc && wxv >= 0.0 && wyv >= 0.0))
    return false;
  *wx = wxv;
  *wy = wyv;
  *height = mx;
  *x = xc;
  *y = yc;
  return true;
}

}  // namespace pose
}  // namespace cp
