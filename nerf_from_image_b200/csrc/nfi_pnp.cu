// Batched PnP pose initialisation (include/nfi_pnp.h, README design 4.12): what the reference's
// compute_pose_pnp gets from OpenCV (SQPnP, the EPnP fallback, iterative LM refinement), one CTA
// per (image, focal guess), all in float64.  oracle/pnp_oracle.py is the same algorithm in numpy.
//
//   compact_kernel  one CTA per image: the foreground pixels' (X, Y, Z, sx, sy), in pixel order
//   solve_kernel    one CTA per (image, focal): per-point sums as block reductions in a fixed
//                   order; the small algebra (Jacobi eigendecompositions, polar factors, the SQP
//                   KKT solve, the LM's 6x6 solve) on thread 0 in local memory
//   select_kernel   one thread per image: the guess with the strictly smallest error, world2cam
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "nfi_check.h"
#include "nfi_pnp.h"

namespace nfi {
namespace pnp {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kPt = 5;          // X, Y, Z, sx, sy
constexpr int kRec = NFI_PNP_RECORD_DOUBLES;
constexpr int kMaxSols = 18;
constexpr int kMaxTerms = 40;
constexpr double kFltEps = 1.1920928955078125e-07;
constexpr double kDblEps = 2.220446049250313e-16;
// SQPnP's constants
constexpr double kRankTol = 1e-7, kSqpSqTol = 1e-10, kSqpDet = 1.001, kOrthoSqErr = 1e-8;
constexpr double kEqVecSq = 1e-10, kEqErrSq = 1e-6, kPointVar = 1e-5;
constexpr int kSqpMaxIter = 15, kLmMaxIter = 20;

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct Shared {
  double red[kWarps][kMaxTerms];
  double out[kMaxTerms];
  double R[9], t[3], jl[9];   // the pose (and LM's left Jacobian) of the current per-point pass
  double A[9], c0[3];         // EPnP: barycentric map alpha_1..3 = A (X - c0)
  double ccs[12];
  double sol_r[kMaxSols][9], sol_t[kMaxSols][3];
  double rvec[3], tvec[3], err, param[6], prev[6];
  double scratch[225];        // thread 0's largest work array: SQP's 15x15 KKT, EPnP's 12x12 M^T M
  int nsol, solver, flag;
};

// sum over the n points of term(point) -> out[0..K): per-thread strided partials, a butterfly
// per warp, then the warps in order
template <int K, class F>
__device__ void block_sum(Shared& s, const double* pts, int n, F term) {
  double acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k] = 0.0;
  for (int i = threadIdx.x; i < n; i += kThreads) {
    double v[K];
    term(pts + (size_t)i * kPt, v);
#pragma unroll
    for (int k = 0; k < K; ++k) acc[k] += v[k];
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const double w = warp_sum_d(acc[k]);
    if (lane == 0) s.red[warp][k] = w;
  }
  __syncthreads();
  if (threadIdx.x < K) {
    double v = 0.0;
    for (int w = 0; w < kWarps; ++w) v += s.red[w][threadIdx.x];
    s.out[threadIdx.x] = v;
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// small algebra (thread 0)
// ------------------------------------------------------------------------------------------------

// eigenvalues w (descending) and eigenvectors (columns of v, row-major n x n, n <= 9) of the
// symmetric a (destroyed) by cyclic Jacobi: rotate while |a_pq| > eps sqrt(|a_pp a_qq|)
__device__ void jacobi_eigh(double* a, int n, double* w, double* v) {
  double u[81];
  for (int i = 0; i < n * n; ++i) u[i] = (i / n == i % n) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 60; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < n - 1; ++p)
      for (int q = p + 1; q < n; ++q) {
        const double apq = a[p * n + q];
        if (apq == 0.0 || fabs(apq) <= kDblEps * sqrt(fabs(a[p * n + p] * a[q * n + q]))) continue;
        rotated = true;
        const double theta = (a[q * n + q] - a[p * n + p]) / (2.0 * apq);
        double t = 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
        if (theta < 0) t = -t;
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < n; ++k) {
          const double akp = a[k * n + p], akq = a[k * n + q];
          a[k * n + p] = c * akp - s * akq;
          a[k * n + q] = s * akp + c * akq;
        }
        for (int k = 0; k < n; ++k) {
          const double apk = a[p * n + k], aqk = a[q * n + k];
          a[p * n + k] = c * apk - s * aqk;
          a[q * n + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < n; ++k) {
          const double ukp = u[k * n + p], ukq = u[k * n + q];
          u[k * n + p] = c * ukp - s * ukq;
          u[k * n + q] = s * ukp + c * ukq;
        }
      }
    if (!rotated) break;
  }
  // stable descending order
  int order[9];
  for (int i = 0; i < n; ++i) order[i] = i;
  for (int i = 1; i < n; ++i) {
    const int o = order[i];
    int j = i;
    while (j > 0 && a[order[j - 1] * n + order[j - 1]] < a[o * n + o]) { order[j] = order[j - 1]; --j; }
    order[j] = o;
  }
  for (int i = 0; i < n; ++i) {
    w[i] = a[order[i] * n + order[i]];
    for (int k = 0; k < n; ++k) v[k * n + i] = u[k * n + order[i]];
  }
}

// singular values (descending) of the symmetric positive semi-definite n x n at, and its left
// singular vectors left in at's rows: one-sided (Hestenes) Jacobi on the rows, each pair rotated
// until orthogonal, up to max(n, 30) sweeps, then sorted by norm and normalised.  EPnP's control
// points depend on these vectors' signs; these are the signs cv2.SVDecomp gives.
__device__ void svd_psd(double* at, int n, double* sig) {
  for (int i = 0; i < n; ++i) {
    double v = 0.0;
    for (int k = 0; k < n; ++k) v += at[i * n + k] * at[i * n + k];
    sig[i] = v;
  }
  const int sweeps = n > 30 ? n : 30;
  for (int it = 0; it < sweeps; ++it) {
    bool changed = false;
    for (int i = 0; i < n - 1; ++i)
      for (int j = i + 1; j < n; ++j) {
        double* ai = at + i * n;
        double* aj = at + j * n;
        double p = 0.0;
        for (int k = 0; k < n; ++k) p += ai[k] * aj[k];
        if (fabs(p) <= kDblEps * sqrt(sig[i] * sig[j])) continue;
        p *= 2;
        const double beta = sig[i] - sig[j], gamma = hypot(p, beta);
        double c, sn;
        if (beta < 0) {
          sn = sqrt((gamma - beta) * 0.5 / gamma);
          c = p / (gamma * sn * 2);
        } else {
          c = sqrt((gamma + beta) / (gamma * 2));
          sn = p / (gamma * c * 2);
        }
        double a = 0.0, b = 0.0;
        for (int k = 0; k < n; ++k) {
          const double t0 = c * ai[k] + sn * aj[k], t1 = -sn * ai[k] + c * aj[k];
          ai[k] = t0, aj[k] = t1;
          a += t0 * t0, b += t1 * t1;
        }
        sig[i] = a, sig[j] = b;
        changed = true;
      }
    if (!changed) break;
  }
  for (int i = 0; i < n; ++i) {
    double v = 0.0;
    for (int k = 0; k < n; ++k) v += at[i * n + k] * at[i * n + k];
    sig[i] = sqrt(v);
  }
  for (int i = 0; i < n - 1; ++i) {
    int j = i;
    for (int k = i + 1; k < n; ++k)
      if (sig[j] < sig[k]) j = k;
    if (j != i) {
      const double t = sig[i]; sig[i] = sig[j]; sig[j] = t;
      for (int k = 0; k < n; ++k) { const double u = at[i * n + k]; at[i * n + k] = at[j * n + k]; at[j * n + k] = u; }
    }
  }
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < n; ++k) at[i * n + k] /= sig[i];
}

__device__ __forceinline__ double det3(const double* m) {
  return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) +
         m[2] * (m[3] * m[7] - m[4] * m[6]);
}

__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// orthogonal factor U V^T of the 3x3 a = U S V^T (proper: the nearest rotation)
__device__ void polar3(const double* a, bool proper, double* out) {
  double ata[9], w[3], v[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) ata[i * 3 + j] = a[i] * a[j] + a[3 + i] * a[3 + j] + a[6 + i] * a[6 + j];
  jacobi_eigh(ata, 3, w, v);
  const double v0[3] = {v[0], v[3], v[6]}, v1[3] = {v[1], v[4], v[7]};
  double u0[3], u1[3], u2[3], v2[3];
  const double inv0 = 1.0 / sqrt(w[0]);
  for (int i = 0; i < 3; ++i) {
    u0[i] = (a[i * 3] * v0[0] + a[i * 3 + 1] * v0[1] + a[i * 3 + 2] * v0[2]) * inv0;
    u1[i] = a[i * 3] * v1[0] + a[i * 3 + 1] * v1[1] + a[i * 3 + 2] * v1[2];
  }
  const double d = u1[0] * u0[0] + u1[1] * u0[1] + u1[2] * u0[2];
  for (int i = 0; i < 3; ++i) u1[i] -= d * u0[i];
  const double inv1 = 1.0 / sqrt(u1[0] * u1[0] + u1[1] * u1[1] + u1[2] * u1[2]);
  for (int i = 0; i < 3; ++i) u1[i] *= inv1;
  cross3(u0, u1, u2);
  cross3(v0, v1, v2);
  const double sign = (proper || det3(a) >= 0) ? 1.0 : -1.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) out[i * 3 + j] = u0[i] * v0[j] + u1[i] * v1[j] + sign * u2[i] * v2[j];
}

__device__ void rodrigues(const double* r, double* R) {
  const double th = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
  if (th < kDblEps) {
    for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    return;
  }
  const double k[3] = {r[0] / th, r[1] / th, r[2] / th};
  const double c = cos(th), s = sin(th), c1 = 1 - c;
  R[0] = c + c1 * k[0] * k[0];        R[1] = c1 * k[0] * k[1] - s * k[2]; R[2] = c1 * k[0] * k[2] + s * k[1];
  R[3] = c1 * k[1] * k[0] + s * k[2]; R[4] = c + c1 * k[1] * k[1];        R[5] = c1 * k[1] * k[2] - s * k[0];
  R[6] = c1 * k[2] * k[0] - s * k[1]; R[7] = c1 * k[2] * k[1] + s * k[0]; R[8] = c + c1 * k[2] * k[2];
}

// axis-angle of m after projecting it on the orthogonal matrices (as cv2.Rodrigues does)
__device__ void rodrigues_inv(const double* m, double* out) {
  double r[9];
  polar3(m, false, r);
  double v[3] = {r[7] - r[5], r[2] - r[6], r[3] - r[1]};
  const double s = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]) * 0.5;
  const double c = fmin(fmax((r[0] + r[4] + r[8] - 1) * 0.5, -1.0), 1.0);
  const double th = acos(c);
  if (s < 1e-5) {
    if (c > 0) {
      out[0] = out[1] = out[2] = 0.0;
      return;
    }
    const double rx = sqrt(fmax((r[0] + 1) * 0.5, 0.0));
    const double ry = sqrt(fmax((r[4] + 1) * 0.5, 0.0)) * (r[1] < 0 ? -1.0 : 1.0);
    double rz = sqrt(fmax((r[8] + 1) * 0.5, 0.0)) * (r[2] < 0 ? -1.0 : 1.0);
    if (fabs(rx) < fabs(ry) && fabs(rx) < fabs(rz) && ((r[5] > 0) != (ry * rz > 0))) rz = -rz;
    const double f = th / sqrt(rx * rx + ry * ry + rz * rz);
    out[0] = rx * f, out[1] = ry * f, out[2] = rz * f;
    return;
  }
  const double f = th / (2.0 * s);
  out[0] = v[0] * f, out[1] = v[1] * f, out[2] = v[2] * f;
}

// J_l(r), the left Jacobian of SO(3): d(R(r) X)/dr = -[R X]x J_l
__device__ void left_jacobian(const double* r, double* jl) {
  const double th2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2], th = sqrt(th2);
  double a, b;
  if (th < 1e-5) {
    a = 0.5, b = 1.0 / 6.0;
  } else {
    a = (1 - cos(th)) / th2, b = (th - sin(th)) / (th2 * th);
  }
  const double k[9] = {0, -r[2], r[1], r[2], 0, -r[0], -r[1], r[0], 0};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double kk = k[i * 3] * k[j] + k[i * 3 + 1] * k[3 + j] + k[i * 3 + 2] * k[6 + j];
      jl[i * 3 + j] = (i == j ? 1.0 : 0.0) + a * k[i * 3 + j] + b * kk;
    }
}

// a x = b (a n x n row-major, destroyed), partial pivoting; x in b; false on a zero pivot
__device__ bool solve_lu(double* a, double* b, int n) {
  for (int k = 0; k < n; ++k) {
    int p = k;
    for (int i = k + 1; i < n; ++i)
      if (fabs(a[i * n + k]) > fabs(a[p * n + k])) p = i;
    if (a[p * n + k] == 0.0) return false;
    if (p != k) {
      for (int j = 0; j < n; ++j) { const double t = a[k * n + j]; a[k * n + j] = a[p * n + j]; a[p * n + j] = t; }
      const double t = b[k]; b[k] = b[p]; b[p] = t;
    }
    for (int i = k + 1; i < n; ++i) {
      const double f = a[i * n + k] / a[k * n + k];
      for (int j = k; j < n; ++j) a[i * n + j] -= f * a[k * n + j];
      b[i] -= f * b[k];
    }
  }
  for (int i = n - 1; i >= 0; --i) {
    double v = b[i];
    for (int j = i + 1; j < n; ++j) v -= a[i * n + j] * b[j];
    b[i] = v / a[i * n + i];
  }
  return true;
}

// least squares of the m x n a (row-major, destroyed) x = b (destroyed), Householder QR
__device__ void lstsq_hh(double* a, int m, int n, double* b, double* x) {
  for (int k = 0; k < n; ++k) {
    double nrm = 0.0;
    for (int i = k; i < m; ++i) nrm += a[i * n + k] * a[i * n + k];
    nrm = sqrt(nrm);
    if (nrm == 0.0) continue;
    const double alpha = a[k * n + k] >= 0 ? -nrm : nrm;
    double v[6];
    for (int i = k; i < m; ++i) v[i - k] = a[i * n + k];
    v[0] -= alpha;
    double vv = 0.0;
    for (int i = 0; i < m - k; ++i) vv += v[i] * v[i];
    if (vv == 0.0) continue;
    for (int j = k; j < n; ++j) {
      double d = 0.0;
      for (int i = k; i < m; ++i) d += v[i - k] * a[i * n + j];
      const double f = 2.0 * d / vv;
      for (int i = k; i < m; ++i) a[i * n + j] -= f * v[i - k];
    }
    double d = 0.0;
    for (int i = k; i < m; ++i) d += v[i - k] * b[i];
    const double f = 2.0 * d / vv;
    for (int i = k; i < m; ++i) b[i] -= f * v[i - k];
  }
  for (int i = n - 1; i >= 0; --i) {
    double v = b[i];
    for (int j = i + 1; j < n; ++j) v -= a[i * n + j] * x[j];
    x[i] = v / a[i * n + i];
  }
}

// ------------------------------------------------------------------------------------------------
// SQPnP (thread 0)
// ------------------------------------------------------------------------------------------------

struct Sqp {
  double omega[81], P[27], mean[3];
  double* kkt;   // [225] in shared memory
  const double* pts;
  int n;
};

// one SQP step from r: min (r+d)^T Omega (r+d) s.t. the linearised row orthonormality (KKT 15x15)
__device__ bool sqp_step(const Sqp& q, const double* r, double* d) {
  double* kkt = q.kkt;
  double rhs[15];
  for (int i = 0; i < 225; ++i) kkt[i] = 0.0;
  for (int i = 0; i < 9; ++i)
    for (int j = 0; j < 9; ++j) kkt[i * 15 + j] = q.omega[i * 9 + j];
  double jac[54];
  for (int i = 0; i < 54; ++i) jac[i] = 0.0;
  const double *r1 = r, *r2 = r + 3, *r3 = r + 6;
  for (int k = 0; k < 3; ++k) {
    jac[0 * 9 + k] = 2 * r1[k];
    jac[1 * 9 + 3 + k] = 2 * r2[k];
    jac[2 * 9 + 6 + k] = 2 * r3[k];
    jac[3 * 9 + k] = r2[k], jac[3 * 9 + 3 + k] = r1[k];
    jac[4 * 9 + 3 + k] = r3[k], jac[4 * 9 + 6 + k] = r2[k];
    jac[5 * 9 + k] = r3[k], jac[5 * 9 + 6 + k] = r1[k];
  }
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 9; ++j) kkt[j * 15 + 9 + i] = kkt[(9 + i) * 15 + j] = jac[i * 9 + j];
  auto dot = [](const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; };
  for (int i = 0; i < 9; ++i) {
    double v = 0.0;
    for (int j = 0; j < 9; ++j) v += q.omega[i * 9 + j] * r[j];
    rhs[i] = -v;
  }
  rhs[9] = 1 - dot(r1, r1), rhs[10] = 1 - dot(r2, r2), rhs[11] = 1 - dot(r3, r3);
  rhs[12] = -dot(r1, r2), rhs[13] = -dot(r2, r3), rhs[14] = -dot(r1, r3);
  if (!solve_lu(kkt, rhs, 15)) return false;
  for (int i = 0; i < 9; ++i) d[i] = rhs[i];
  return true;
}

__device__ void run_sqp(const Sqp& q, const double* r0, double* out) {
  double r[9], d[9];
  for (int i = 0; i < 9; ++i) r[i] = r0[i];
  for (int it = 0; it < kSqpMaxIter; ++it) {
    if (!sqp_step(q, r, d)) break;
    double dd = 0.0;
    for (int i = 0; i < 9; ++i) r[i] += d[i], dd += d[i] * d[i];
    if (dd <= kSqpSqTol) break;
  }
  double dr = det3(r);
  if (dr < 0) {
    for (int i = 0; i < 9; ++i) r[i] = -r[i];
    dr = -dr;
  }
  if (dr > kSqpDet)
    polar3(r, true, out);
  else
    for (int i = 0; i < 9; ++i) out[i] = r[i];
}

struct SqpBest {
  double min_err;
  double err[kMaxSols];
};

__device__ void sqp_check(const Sqp& q, Shared& s, SqpBest& b, const double* r) {
  double t[3];
  for (int i = 0; i < 3; ++i) {
    double v = 0.0;
    for (int j = 0; j < 9; ++j) v += q.P[i * 9 + j] * r[j];
    t[i] = v;
  }
  bool front = r[6] * q.mean[0] + r[7] * q.mean[1] + r[8] * q.mean[2] + t[2] > 0;
  if (!front) {  // the majority of the points then
    int npos = 0;
    for (int i = 0; i < q.n; ++i) {
      const double* p = q.pts + (size_t)i * kPt;
      npos += (r[6] * p[0] + r[7] * p[1] + r[8] * p[2] + t[2]) > 0;
    }
    front = npos >= q.n - npos;
  }
  if (!front) return;
  double err = 0.0;
  for (int i = 0; i < 9; ++i) {
    double v = 0.0;
    for (int j = 0; j < 9; ++j) v += q.omega[i * 9 + j] * r[j];
    err += r[i] * v;
  }
  auto put = [&](int k) {
    for (int i = 0; i < 9; ++i) s.sol_r[k][i] = r[i];
    for (int i = 0; i < 3; ++i) s.sol_t[k][i] = t[i];
    b.err[k] = err;
  };
  if (fabs(b.min_err - err) > kEqErrSq) {
    if (b.min_err > err) {
      b.min_err = err;
      put(0);
      s.nsol = 1;
    }
    return;
  }
  bool found = false;
  for (int k = 0; k < s.nsol; ++k) {
    double dd = 0.0;
    for (int i = 0; i < 9; ++i) dd += (s.sol_r[k][i] - r[i]) * (s.sol_r[k][i] - r[i]);
    if (dd < kEqVecSq) {
      if (b.err[k] > err) put(k);
      found = true;
      break;
    }
  }
  if (!found && s.nsol < kMaxSols) put(s.nsol++);
  if (b.min_err > err) b.min_err = err;
}

__device__ void sqp_both_signs(const Sqp& q, Shared& s, SqpBest& b, const double* e) {
  double r0[9], r[9], m[9];
  for (int sign = 0; sign < 2; ++sign) {
    for (int i = 0; i < 9; ++i) m[i] = sign ? -e[i] : e[i];
    polar3(m, true, r0);
    run_sqp(q, r0, r);
    sqp_check(q, s, b, r);
  }
}

// the 39 sums: S0, Sx, Sy, Ss (sum w X X^T upper, 6 each), sX, sxX, syX, ssX (3 each), sx, sy, ss
__device__ void sqpnp_terms(const double* p, double inv_f, double* v) {
  const double x = p[3] * inv_f, y = p[4] * inv_f, sq = x * x + y * y;
  const double xx[6] = {p[0] * p[0], p[0] * p[1], p[0] * p[2], p[1] * p[1], p[1] * p[2], p[2] * p[2]};
  for (int k = 0; k < 6; ++k) v[k] = xx[k], v[6 + k] = x * xx[k], v[12 + k] = y * xx[k], v[18 + k] = sq * xx[k];
  for (int k = 0; k < 3; ++k) v[24 + k] = p[k], v[27 + k] = x * p[k], v[30 + k] = y * p[k], v[33 + k] = sq * p[k];
  v[36] = x, v[37] = y, v[38] = sq;
}

// thread 0: from the sums, the SQPnP solutions into s.sol_*, s.nsol; -1 when the image points
// have too little spread
__device__ void sqpnp_solve(Shared& s, const double* sums, const double* pts, int n) {
  Sqp q;
  q.pts = pts, q.n = n, q.kkt = s.scratch;
  auto sym = [](const double* u, int i, int j) {  // the upper triangle of a symmetric 3x3
    const int idx[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
    return u[idx[i][j]];
  };
  for (int i = 0; i < 81; ++i) q.omega[i] = 0.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double s0 = sym(sums, i, j), sx = sym(sums + 6, i, j), sy = sym(sums + 12, i, j),
                   ss = sym(sums + 18, i, j);
      q.omega[i * 9 + j] = s0;
      q.omega[(3 + i) * 9 + 3 + j] = s0;
      q.omega[i * 9 + 6 + j] = -sx;
      q.omega[(3 + i) * 9 + 6 + j] = -sy;
      q.omega[(6 + i) * 9 + j] = -sx;
      q.omega[(6 + i) * 9 + 3 + j] = -sy;
      q.omega[(6 + i) * 9 + 6 + j] = ss;
    }
  const double *sX = sums + 24, *sxX = sums + 27, *syX = sums + 30, *ssX = sums + 33;
  const double sx = sums[36], sy = sums[37], ss = sums[38], dn = (double)n;
  double qa[27];
  for (int i = 0; i < 27; ++i) qa[i] = 0.0;
  for (int k = 0; k < 3; ++k) {
    qa[0 * 9 + k] = sX[k], qa[0 * 9 + 6 + k] = -sxX[k];
    qa[1 * 9 + 3 + k] = sX[k], qa[1 * 9 + 6 + k] = -syX[k];
    qa[2 * 9 + k] = -sxX[k], qa[2 * 9 + 3 + k] = -syX[k], qa[2 * 9 + 6 + k] = ssX[k];
  }
  const double qm[9] = {dn, 0, -sx, 0, dn, -sy, -sx, -sy, ss};
  const double detq = dn * (dn * ss - sy * sy - sx * sx);
  if (detq / (dn * dn * dn) < kPointVar) {
    s.nsol = -1;
    return;
  }
  const double qi[9] = {(qm[4] * qm[8] - qm[5] * qm[7]) / detq, (qm[2] * qm[7] - qm[1] * qm[8]) / detq,
                        (qm[1] * qm[5] - qm[2] * qm[4]) / detq, (qm[5] * qm[6] - qm[3] * qm[8]) / detq,
                        (qm[0] * qm[8] - qm[2] * qm[6]) / detq, (qm[2] * qm[3] - qm[0] * qm[5]) / detq,
                        (qm[3] * qm[7] - qm[4] * qm[6]) / detq, (qm[1] * qm[6] - qm[0] * qm[7]) / detq,
                        (qm[0] * qm[4] - qm[1] * qm[3]) / detq};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 9; ++j)
      q.P[i * 9 + j] = -(qi[i * 3] * qa[j] + qi[i * 3 + 1] * qa[9 + j] + qi[i * 3 + 2] * qa[18 + j]);
  for (int i = 0; i < 9; ++i)
    for (int j = 0; j < 9; ++j)
      q.omega[i * 9 + j] += qa[i] * q.P[j] + qa[9 + i] * q.P[9 + j] + qa[18 + i] * q.P[18 + j];
  for (int k = 0; k < 3; ++k) q.mean[k] = sX[k] / dn;
  double a[81], w[9], u[81];
  for (int i = 0; i < 81; ++i) a[i] = q.omega[i];
  jacobi_eigh(a, 9, w, u);
  int nnull = 0;
  while (nnull < 8 && w[7 - nnull] < kRankTol) ++nnull;
  const int neig = nnull > 0 ? nnull : 1;
  SqpBest b;
  b.min_err = INFINITY;
  s.nsol = 0;
  double e[9];
  for (int i = 9 - neig; i < 9; ++i) {
    for (int k = 0; k < 9; ++k) e[k] = sqrt(3.0) * u[k * 9 + i];
    double oe = 0.0;
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        const double d = e[r * 3] * e[c * 3] + e[r * 3 + 1] * e[c * 3 + 1] + e[r * 3 + 2] * e[c * 3 + 2] -
                         (r == c ? 1.0 : 0.0);
        oe += d * d;
      }
    if (oe < kOrthoSqErr) {
      const double de = det3(e);
      for (int k = 0; k < 9; ++k) e[k] *= de;
      sqp_check(q, s, b, e);
    } else {
      sqp_both_signs(q, s, b, e);
    }
  }
  for (int c = 1; 9 - neig - c > 0 && b.min_err > 3 * w[9 - neig - c]; ++c) {
    for (int k = 0; k < 9; ++k) e[k] = u[k * 9 + 9 - neig - c];
    sqp_both_signs(q, s, b, e);
  }
}

// ------------------------------------------------------------------------------------------------
// per-point terms
// ------------------------------------------------------------------------------------------------

struct ProjSq {  // |proj - screen|^2
  const double *R, *t;
  double f;
  __device__ void operator()(const double* p, double* v) const {
    const double x = R[0] * p[0] + R[1] * p[1] + R[2] * p[2] + t[0];
    const double y = R[3] * p[0] + R[4] * p[1] + R[5] * p[2] + t[1];
    const double z = R[6] * p[0] + R[7] * p[1] + R[8] * p[2] + t[2];
    const double iz = 1.0 / z, dx = f * x * iz - p[3], dy = f * y * iz - p[4];
    v[0] = dx * dx + dy * dy;
  }
};

struct ProjDist {  // |proj - screen| (EPnP's own choice among its approximations)
  const double *R, *t;
  double f;
  __device__ void operator()(const double* p, double* v) const {
    ProjSq{R, t, f}(p, v);
    v[0] = sqrt(v[0]);
  }
};

// LM: J^T J (upper, 21), J^T r (6), |r|^2 at the pose (R, t) with rvec's left Jacobian jl
struct LmTerms {
  const double *R, *t, *jl;
  double f;
  __device__ void operator()(const double* p, double* v) const {
    double pw[3], pc[3];
    for (int i = 0; i < 3; ++i) pw[i] = R[i * 3] * p[0] + R[i * 3 + 1] * p[1] + R[i * 3 + 2] * p[2], pc[i] = pw[i] + t[i];
    const double iz = 1.0 / pc[2];
    const double r0 = f * pc[0] * iz - p[3], r1 = f * pc[1] * iz - p[4];
    const double dp[2][3] = {{f * iz, 0.0, -f * pc[0] * iz * iz}, {0.0, f * iz, -f * pc[1] * iz * iz}};
    double J[2][6];
    for (int k = 0; k < 3; ++k) {
      const double col[3] = {jl[k], jl[3 + k], jl[6 + k]};
      double d[3];
      cross3(col, pw, d);
      for (int r = 0; r < 2; ++r) J[r][k] = dp[r][0] * d[0] + dp[r][1] * d[1] + dp[r][2] * d[2], J[r][3 + k] = dp[r][k];
    }
    int o = 0;
    for (int i = 0; i < 6; ++i)
      for (int j = i; j < 6; ++j) v[o++] = J[0][i] * J[0][j] + J[1][i] * J[1][j];
    for (int i = 0; i < 6; ++i) v[21 + i] = J[0][i] * r0 + J[1][i] * r1;
    v[27] = r0 * r0 + r1 * r1;
  }
};

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kThreads) compact_kernel(nfi_pnp_params p, double* pts, int* count) {
  const int b = blockIdx.x, HW = p.height * p.width;
  const uint8_t* m = p.mask + (size_t)b * HW;
  double* out = pts + (size_t)b * HW * kPt;
  __shared__ int warp_n[kWarps];
  __shared__ int base;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c0 = 0; c0 < HW; c0 += kThreads) {
    const int i = c0 + threadIdx.x;
    const bool fg = i < HW && m[i] != 0;
    const unsigned ball = __ballot_sync(0xffffffffu, fg);
    if (lane == 0) warp_n[warp] = __popc(ball);
    __syncthreads();
    int off = base;
    for (int w = 0; w < warp; ++w) off += warp_n[w];
    off += __popc(ball & ((1u << lane) - 1u));
    if (fg) {
      const int y = i / p.width, x = i % p.width;
      const float* c = p.coords + b * p.coords_stride[0] + y * p.coords_stride[1] + x * p.coords_stride[2];
      double* o = out + (size_t)off * kPt;
      o[0] = (double)c[0];
      o[1] = (double)c[p.coords_stride[3]];
      o[2] = (double)c[2 * p.coords_stride[3]];
      o[3] = (double)x / p.width - 0.5;
      o[4] = (double)y / p.height - 0.5;
    }
    __syncthreads();
    if (threadIdx.x == 0)
      for (int w = 0; w < kWarps; ++w) base += warp_n[w];
    __syncthreads();
  }
  if (threadIdx.x == 0) count[b] = base;
}

// thread 0: rvec of the 3x3 M, and the R(rvec) and t the per-point passes use
__device__ void set_pose(Shared& s, const double* M, const double* t) {
  rodrigues_inv(M, s.rvec);
  rodrigues(s.rvec, s.R);
  for (int i = 0; i < 3; ++i) s.t[i] = t[i], s.tvec[i] = t[i];
}

__device__ void epnp_ccs_pose(Shared& s, const double* alpha0, const double* ccs, const double* sa,
                              const double* sad, int n, double* R, double* t) {
  // sign: the first point in front of the camera
  double z0 = 0.0, sg = 1.0;
  for (int j = 0; j < 4; ++j) z0 += alpha0[j] * ccs[3 * j + 2];
  if (z0 < 0) sg = -1.0;
  // pc0 = sum_j mean(alpha_j) ccs_j; ABt = sum_j ccs_j (sum_i alpha_ij (X_i - c0))^T
  double pc0[3] = {0, 0, 0}, abt[9];
  for (int j = 0; j < 4; ++j)
    for (int k = 0; k < 3; ++k) pc0[k] += sg * sa[j] / n * ccs[3 * j + k];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double v = 0.0;
      for (int j = 0; j < 4; ++j) v += sg * ccs[3 * j + r] * sad[3 * j + c];
      abt[r * 3 + c] = v;
    }
  polar3(abt, false, R);
  if (det3(R) < 0)
    for (int k = 0; k < 3; ++k) R[6 + k] = -R[6 + k];
  for (int i = 0; i < 3; ++i) t[i] = pc0[i] - (R[i * 3] * s.c0[0] + R[i * 3 + 1] * s.c0[1] + R[i * 3 + 2] * s.c0[2]);
}

__global__ void __launch_bounds__(kThreads) solve_kernel(nfi_pnp_params p, const double* all_pts,
                                                         const int* count, double* cand_out) {
  __shared__ Shared s;
  const int b = blockIdx.x / p.n_focals, fi = blockIdx.x % p.n_focals;
  const int n = count[b];
  const double* pts = all_pts + (size_t)b * p.height * p.width * kPt;
  double* cand = cand_out + (size_t)blockIdx.x * kRec;
  const int tid = threadIdx.x;
  if (n < 4) {
    if (tid < kRec) cand[tid] = 0.0;
    return;
  }
  const double f = p.focals[fi], inv_f = 1.0 / f;

  // ---- SQPnP
  block_sum<39>(s, pts, n, [&](const double* q, double* v) { sqpnp_terms(q, inv_f, v); });
  if (tid == 0) {
    double sums[39];
    for (int k = 0; k < 39; ++k) sums[k] = s.out[k];
    sqpnp_solve(s, sums, pts, n);
    s.solver = 0;
    s.err = INFINITY;
  }
  __syncthreads();
  const int nsol = s.nsol;
  for (int k = 0; k < nsol; ++k) {
    if (tid == 0) {
      double rv[3], R[9];
      rodrigues_inv(s.sol_r[k], rv);
      rodrigues(rv, R);
      for (int i = 0; i < 9; ++i) s.R[i] = R[i];
      for (int i = 0; i < 3; ++i) s.t[i] = s.sol_t[k][i], s.param[i] = rv[i];
    }
    __syncthreads();
    block_sum<1>(s, pts, n, ProjSq{s.R, s.t, f});
    if (tid == 0) {
      const double e = sqrt(s.out[0] / (2.0 * n));
      if (s.t[2] > 0 && (s.solver == 0 || e < s.err)) {
        s.solver = 1, s.err = e;
        for (int i = 0; i < 3; ++i) s.rvec[i] = s.param[i], s.tvec[i] = s.t[i];
      }
    }
    __syncthreads();
  }

  // ---- EPnP
  if (s.solver == 0) {
    block_sum<3>(s, pts, n, [](const double* q, double* v) { v[0] = q[0], v[1] = q[1], v[2] = q[2]; });
    if (tid == 0)
      for (int k = 0; k < 3; ++k) s.c0[k] = s.out[k] / n;
    __syncthreads();
    block_sum<6>(s, pts, n, [&](const double* q, double* v) {
      const double d[3] = {q[0] - s.c0[0], q[1] - s.c0[1], q[2] - s.c0[2]};
      v[0] = d[0] * d[0], v[1] = d[0] * d[1], v[2] = d[0] * d[2], v[3] = d[1] * d[1], v[4] = d[1] * d[2], v[5] = d[2] * d[2];
    });
    if (tid == 0) {
      double a[9] = {s.out[0], s.out[1], s.out[2], s.out[1], s.out[3], s.out[4], s.out[2], s.out[4], s.out[5]};
      double w[3];
      svd_psd(a, 3, w);   // a's rows: the principal axes
      // control points c0 + k_i axis_i; CC (columns k_i axis_i) inverted
      double cc[9];
      for (int c = 0; c < 3; ++c) {
        const double k = sqrt(w[c] / n);
        for (int r = 0; r < 3; ++r) cc[r * 3 + c] = k * a[c * 3 + r];
      }
      const double d = det3(cc);
      s.A[0] = (cc[4] * cc[8] - cc[5] * cc[7]) / d, s.A[1] = (cc[2] * cc[7] - cc[1] * cc[8]) / d;
      s.A[2] = (cc[1] * cc[5] - cc[2] * cc[4]) / d, s.A[3] = (cc[5] * cc[6] - cc[3] * cc[8]) / d;
      s.A[4] = (cc[0] * cc[8] - cc[2] * cc[6]) / d, s.A[5] = (cc[2] * cc[3] - cc[0] * cc[5]) / d;
      s.A[6] = (cc[3] * cc[7] - cc[4] * cc[6]) / d, s.A[7] = (cc[1] * cc[6] - cc[0] * cc[7]) / d;
      s.A[8] = (cc[0] * cc[4] - cc[1] * cc[3]) / d;
      for (int i = 0; i < 9; ++i) s.ccs[i] = cc[i];   // keep CC for rho
    }
    __syncthreads();
    auto alphas = [&](const double* q, double* al) {
      const double d[3] = {q[0] - s.c0[0], q[1] - s.c0[1], q[2] - s.c0[2]};
      for (int j = 0; j < 3; ++j) al[1 + j] = s.A[j * 3] * d[0] + s.A[j * 3 + 1] * d[1] + s.A[j * 3 + 2] * d[2];
      al[0] = 1 - al[1] - al[2] - al[3];
    };
    // sum a_j a_k, a_j a_k u, a_j a_k v, a_j a_k (u^2 + v^2) over the 10 pairs j <= k
    block_sum<40>(s, pts, n, [&](const double* q, double* v) {
      double al[4];
      alphas(q, al);
      const double u = q[3], w = q[4], sq = u * u + w * w;
      int o = 0;
      for (int j = 0; j < 4; ++j)
        for (int k = j; k < 4; ++k, ++o) {
          const double aa = al[j] * al[k];
          v[o] = aa, v[10 + o] = aa * u, v[20 + o] = aa * w, v[30 + o] = aa * sq;
        }
    });
    __shared__ double mstat[40];
    if (tid < 40) mstat[tid] = s.out[tid];
    __syncthreads();
    // sum a_j (X - c0) (12) and sum a_j (4)
    block_sum<16>(s, pts, n, [&](const double* q, double* v) {
      double al[4];
      alphas(q, al);
      for (int j = 0; j < 4; ++j) {
        v[12 + j] = al[j];
        for (int k = 0; k < 3; ++k) v[3 * j + k] = al[j] * (q[k] - s.c0[k]);
      }
    });
    __shared__ double ccs_all[3][12];
    __shared__ double sad[16];
    if (tid < 16) sad[tid] = s.out[tid];
    __syncthreads();
    if (tid == 0) {
      int pair[4][4], o = 0;
      for (int j = 0; j < 4; ++j)
        for (int k = j; k < 4; ++k, ++o) pair[j][k] = pair[k][j] = o;
      double* mtm = s.scratch;
      for (int j = 0; j < 4; ++j)
        for (int k = 0; k < 4; ++k) {
          const int pk = pair[j][k];
          double* blk[3];
          for (int a = 0; a < 3; ++a) blk[a] = mtm + (3 * j + a) * 12 + 3 * k;
          blk[0][0] = f * f * mstat[pk], blk[0][1] = 0.0, blk[0][2] = -f * mstat[10 + pk];
          blk[1][0] = 0.0, blk[1][1] = f * f * mstat[pk], blk[1][2] = -f * mstat[20 + pk];
          blk[2][0] = -f * mstat[10 + pk], blk[2][1] = -f * mstat[20 + pk], blk[2][2] = mstat[30 + pk];
        }
      double w[12];
      svd_psd(mtm, 12, w);
      double nv[4][12];
      for (int k = 0; k < 4; ++k)
        for (int i = 0; i < 12; ++i) nv[k][i] = mtm[(11 - k) * 12 + i];
      // control points in world: c0, c0 + CC columns
      double cws[4][3];
      for (int k = 0; k < 3; ++k) cws[0][k] = s.c0[k];
      for (int j = 1; j < 4; ++j)
        for (int k = 0; k < 3; ++k) cws[j][k] = s.c0[k] + s.ccs[k * 3 + j - 1];
      const int prs[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};
      double L[60], rho[6];
      for (int i = 0; i < 6; ++i) {
        const int a = prs[i][0], c = prs[i][1];
        double dv[4][3];
        for (int k = 0; k < 4; ++k)
          for (int m = 0; m < 3; ++m) dv[k][m] = nv[k][3 * a + m] - nv[k][3 * c + m];
        auto dt = [&](int x, int y) { return dv[x][0] * dv[y][0] + dv[x][1] * dv[y][1] + dv[x][2] * dv[y][2]; };
        double* l = L + i * 10;
        l[0] = dt(0, 0), l[1] = 2 * dt(0, 1), l[2] = dt(1, 1), l[3] = 2 * dt(0, 2), l[4] = 2 * dt(1, 2);
        l[5] = dt(2, 2), l[6] = 2 * dt(0, 3), l[7] = 2 * dt(1, 3), l[8] = 2 * dt(2, 3), l[9] = dt(3, 3);
        double e2 = 0.0;
        for (int m = 0; m < 3; ++m) e2 += (cws[a][m] - cws[c][m]) * (cws[a][m] - cws[c][m]);
        rho[i] = e2;
      }
      double betas[3][4];
      {  // approximation 1: [B11 B12 B13 B14]
        double a[24], rb[6], x[4];
        const int cols[4] = {0, 1, 3, 6};
        for (int i = 0; i < 6; ++i) {
          rb[i] = rho[i];
          for (int c = 0; c < 4; ++c) a[i * 4 + c] = L[i * 10 + cols[c]];
        }
        lstsq_hh(a, 6, 4, rb, x);
        betas[0][0] = sqrt(fabs(x[0]));
        for (int k = 1; k < 4; ++k) betas[0][k] = (x[0] < 0 ? -x[k] : x[k]) / betas[0][0];
      }
      for (int ap = 0; ap < 2; ++ap) {  // approximations 2 ([B11 B12 B22]) and 3 (+ B13 B23)
        const int nc = ap == 0 ? 3 : 5;
        double a[30], rb[6], x[5];
        for (int i = 0; i < 6; ++i) {
          rb[i] = rho[i];
          for (int c = 0; c < nc; ++c) a[i * nc + c] = L[i * 10 + c];
        }
        lstsq_hh(a, 6, nc, rb, x);
        double* bt = betas[1 + ap];
        if (x[0] < 0) {
          bt[0] = sqrt(-x[0]);
          bt[1] = x[2] < 0 ? sqrt(-x[2]) : 0.0;
        } else {
          bt[0] = sqrt(x[0]);
          bt[1] = x[2] > 0 ? sqrt(x[2]) : 0.0;
        }
        if (x[1] < 0) bt[0] = -bt[0];
        bt[2] = ap == 1 ? x[3] / bt[0] : 0.0;
        bt[3] = 0.0;
      }
      for (int c = 0; c < 3; ++c) {  // five Gauss-Newton steps on each
        double* bt = betas[c];
        for (int it = 0; it < 5; ++it) {
          const double b0 = bt[0], b1 = bt[1], b2 = bt[2], b3 = bt[3];
          const double pr[10] = {b0 * b0, b0 * b1, b1 * b1, b0 * b2, b1 * b2, b2 * b2, b0 * b3, b1 * b3, b2 * b3, b3 * b3};
          double a[24], rb[6], x[4];
          for (int i = 0; i < 6; ++i) {
            const double* l = L + i * 10;
            a[i * 4 + 0] = 2 * l[0] * b0 + l[1] * b1 + l[3] * b2 + l[6] * b3;
            a[i * 4 + 1] = l[1] * b0 + 2 * l[2] * b1 + l[4] * b2 + l[7] * b3;
            a[i * 4 + 2] = l[3] * b0 + l[4] * b1 + 2 * l[5] * b2 + l[8] * b3;
            a[i * 4 + 3] = l[6] * b0 + l[7] * b1 + l[8] * b2 + 2 * l[9] * b3;
            double v = 0.0;
            for (int k = 0; k < 10; ++k) v += l[k] * pr[k];
            rb[i] = rho[i] - v;
          }
          lstsq_hh(a, 6, 4, rb, x);
          for (int k = 0; k < 4; ++k) bt[k] += x[k];
        }
        for (int i = 0; i < 12; ++i) {
          double v = 0.0;
          for (int k = 0; k < 4; ++k) v += bt[k] * nv[k][i];
          ccs_all[c][i] = v;
        }
      }
    }
    __syncthreads();
    // the first point's alphas decide each approximation's sign
    __shared__ double alpha0[4];
    if (tid == 0) alphas(pts, alpha0);
    __syncthreads();
    double best_e = INFINITY;
    for (int c = 0; c < 3; ++c) {
      if (tid == 0) epnp_ccs_pose(s, alpha0, ccs_all[c], sad + 12, sad, n, s.R, s.t);
      __syncthreads();
      block_sum<1>(s, pts, n, ProjDist{s.R, s.t, f});
      if (tid == 0 && s.out[0] / n < best_e) {
        best_e = s.out[0] / n;
        for (int i = 0; i < 9; ++i) s.A[i] = s.R[i];
        for (int i = 0; i < 3; ++i) s.param[i] = s.t[i];
      }
      __syncthreads();
    }
    if (tid == 0) set_pose(s, s.A, s.param);
    __syncthreads();
    block_sum<1>(s, pts, n, ProjSq{s.R, s.t, f});
    if (tid == 0 && s.tvec[2] > 0) s.solver = 2, s.err = sqrt(s.out[0] / (2.0 * n));
    __syncthreads();
  }

  // ---- Levenberg-Marquardt
  int accepted = 0;
  if (s.solver != 0 && p.refine) {
    int lam = -3;
    if (tid == 0) {
      for (int i = 0; i < 3; ++i) s.param[i] = s.rvec[i], s.param[3 + i] = s.tvec[i];
      rodrigues(s.param, s.R);
      left_jacobian(s.param, s.jl);
      for (int i = 0; i < 3; ++i) s.t[i] = s.param[3 + i];
    }
    __syncthreads();
    block_sum<28>(s, pts, n, LmTerms{s.R, s.t, s.jl, f});
    double prev_err = sqrt(s.out[27]);  // every thread: same bits
    double jtj[36], jtr[6];
    for (int it = 0; it < kLmMaxIter; ++it) {
      {
        int o = 0;
        for (int i = 0; i < 6; ++i)
          for (int j = i; j < 6; ++j, ++o) jtj[i * 6 + j] = jtj[j * 6 + i] = s.out[o];
        for (int i = 0; i < 6; ++i) jtr[i] = s.out[21 + i];
      }
      __syncthreads();
      if (tid == 0)
        for (int i = 0; i < 6; ++i) s.prev[i] = s.param[i];
      double err;
      for (;;) {
        if (tid == 0) {
          double a[36], x[6];
          for (int i = 0; i < 36; ++i) a[i] = jtj[i];
          const double damp = 1.0 + exp(lam * log(10.0));
          for (int i = 0; i < 6; ++i) a[i * 6 + i] *= damp, x[i] = jtr[i];
          const bool ok = solve_lu(a, x, 6);
          for (int i = 0; i < 6; ++i) s.param[i] = s.prev[i] - (ok ? x[i] : 0.0);
          rodrigues(s.param, s.R);
          for (int i = 0; i < 3; ++i) s.t[i] = s.param[3 + i];
        }
        __syncthreads();
        block_sum<1>(s, pts, n, ProjSq{s.R, s.t, f});
        err = sqrt(s.out[0]);
        if (!(err > prev_err)) break;
        if (++lam > 16) break;
      }
      lam = lam - 1 < -16 ? -16 : lam - 1;
      double dd = 0.0, pp = 0.0;
      for (int i = 0; i < 6; ++i) dd += (s.param[i] - s.prev[i]) * (s.param[i] - s.prev[i]), pp += s.prev[i] * s.prev[i];
      if (it + 1 >= kLmMaxIter || sqrt(dd) < kFltEps * sqrt(pp)) break;
      prev_err = err;
      __syncthreads();
      if (tid == 0) left_jacobian(s.param, s.jl);
      __syncthreads();
      block_sum<28>(s, pts, n, LmTerms{s.R, s.t, s.jl, f});
    }
    if (s.param[5] > 0) {
      accepted = 1;
      block_sum<1>(s, pts, n, ProjSq{s.R, s.t, f});
      if (tid == 0) {
        s.err = sqrt(s.out[0] / (2.0 * n));
        for (int i = 0; i < 3; ++i) s.rvec[i] = s.param[i], s.tvec[i] = s.param[3 + i];
      }
    }
    __syncthreads();
  }
  if (tid == 0) {
    cand[0] = s.solver, cand[1] = accepted;
    for (int i = 0; i < 3; ++i) cand[2 + i] = s.solver ? s.rvec[i] : 0.0, cand[5 + i] = s.solver ? s.tvec[i] : 0.0;
    cand[8] = s.solver ? s.err : 0.0;
  }
}

__global__ void select_kernel(nfi_pnp_params p, const double* cand) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= p.batch) return;
  const int F = p.n_focals;
  int best = -1;
  for (int f = 0; f < F; ++f) {
    const double* c = cand + ((size_t)b * F + f) * kRec;
    if (c[0] != 0.0 && (best < 0 || c[8] < cand[((size_t)b * F + best) * kRec + 8])) best = f;
  }
  double rv[3] = {0, 0, 0}, t[3] = {0, 0, -10}, focal = 1.0, err = 10.0, R[9];
  if (best >= 0) {
    const double* c = cand + ((size_t)b * F + best) * kRec;
    for (int i = 0; i < 3; ++i) rv[i] = c[2 + i], t[i] = c[5 + i];
    focal = p.focals[best], err = c[8];
  }
  rodrigues(rv, R);
  double* m = p.world2cam + (size_t)b * 16;
  for (int i = 0; i < 3; ++i) {
    const double sg = i == 0 ? 1.0 : -1.0;
    for (int j = 0; j < 3; ++j) m[i * 4 + j] = sg * R[i * 3 + j];
    m[i * 4 + 3] = sg * t[i];
  }
  m[12] = m[13] = m[14] = 0.0, m[15] = 1.0;
  p.focal[b] = focal;
  p.error[b] = err;
  if (p.record)
    for (int i = 0; i < F * kRec; ++i) p.record[(size_t)b * F * kRec + i] = cand[(size_t)b * F * kRec + i];
}

struct Layout {
  size_t pts, cand, count, total;
};

Layout layout(const nfi_pnp_params& p) {
  auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
  Layout l;
  l.pts = 0;
  l.cand = up((size_t)p.batch * p.height * p.width * kPt * sizeof(double));
  l.count = l.cand + up((size_t)p.batch * p.n_focals * kRec * sizeof(double));
  l.total = l.count + up((size_t)p.batch * sizeof(int));
  return l;
}

int check(const nfi_pnp_params* p) {
  if (p == nullptr) return fail("params is NULL");
  if (p->batch <= 0 || p->height <= 0 || p->width <= 0) return fail("pnp: empty batch or image");
  if ((int64_t)p->height * p->width > (1 << 24)) return fail("pnp: more than 2^24 pixels per image");
  if (p->n_focals < 1 || p->n_focals > NFI_PNP_MAX_FOCALS)
    return fail("pnp: n_focals must be 1..%d, got %d", NFI_PNP_MAX_FOCALS, p->n_focals);
  if (p->refine != 0 && p->refine != 1) return fail("pnp: refine must be 0 or 1");
  return 0;
}

}  // namespace
}  // namespace pnp
}  // namespace nfi

extern "C" {

size_t nfi_pnp_workspace_bytes(const nfi_pnp_params* params) {
  if (nfi::pnp::check(params)) return 0;
  return nfi::pnp::layout(*params).total;
}

int nfi_pnp_solve(const nfi_pnp_params* params, void* stream) {
  using namespace nfi::pnp;
  if (const int rc = check(params)) return rc;
  const nfi_pnp_params& p = *params;
  if (!p.coords || !p.mask || !p.focals || !p.world2cam || !p.focal || !p.error || !p.workspace)
    return nfi::fail("pnp: coords, mask, focals, the outputs and the workspace must be given");
  const Layout l = layout(p);
  if (p.workspace_bytes < l.total)
    return nfi::fail("pnp: workspace too small (%zu < %zu bytes)", p.workspace_bytes, l.total);
  char* ws = (char*)p.workspace;
  double* pts = (double*)(ws + l.pts);
  double* cand = (double*)(ws + l.cand);
  int* count = (int*)(ws + l.count);
  cudaStream_t s = (cudaStream_t)stream;
  compact_kernel<<<p.batch, kThreads, 0, s>>>(p, pts, count);
  NFI_CUDA(cudaGetLastError());
  solve_kernel<<<p.batch * p.n_focals, kThreads, 0, s>>>(p, pts, count, cand);
  NFI_CUDA(cudaGetLastError());
  select_kernel<<<(p.batch + 63) / 64, 64, 0, s>>>(p, cand);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
