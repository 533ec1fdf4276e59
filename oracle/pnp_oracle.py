"""Float64 restatement of the reference's PnP pose initialisation (lib/pose_estimation.py::
compute_pose_pnp), step for step as nerf_from_image_b200/csrc/nfi_pnp.cu does it.

The reference calls OpenCV: SQPnP (Terzakis & Lourakis, ECCV 2020), EPnP (Lepetit, Moreno-Noguer &
Fua, IJCV 2009) where SQPnP gives no pose in front of the camera, and then OpenCV's iterative
Levenberg-Marquardt refinement.  Each is written here from its paper and from what cv2 returns:

- SQPnP: the 9x9 matrix Omega of the algebraic error sum_i |A_i (R X_i + t)|^2 with
  A_i = [[1, 0, -x], [0, 1, -y]] on normalised image points, t eliminated in closed form; SQP from
  the nearest rotations of the eigenvectors of the smallest eigenvalues, kept when the centroid (or
  else the majority of points) lies in front of the camera.
- EPnP: four control points on the principal axes of the points (signs as cv2's SVD gives them), the 12x12 M^T M, the three
  beta approximations refined by five Gauss-Newton steps on the control-point distances, and the
  one with the smallest mean reprojection distance.
- LM on (Rodrigues rvec, t): multiplicative damping diag(J^T J) (1 + 10^k), k from -3, up one on a
  rejected step (up to 16), down one (to -16) after each iteration; at most 20 iterations, stopping
  when |dp| / |p| < FLT_EPSILON.

The small algebra (symmetric Jacobi eigendecomposition, polar factors, Householder least squares,
the LM's 6x6 solve) is the same code path as the kernels'; numpy only does the per-point sums.
"""
import math

import numpy as np

FLT_EPSILON = 1.1920928955078125e-07
DBL_EPSILON = 2.220446049250313e-16
SOLVER_NONE, SOLVER_SQPNP, SOLVER_EPNP = 0, 1, 2
MAX_SQPNP_SOLUTIONS = 18

# SQPnP's constants (the paper's implementation and OpenCV use the same values)
RANK_TOLERANCE = 1e-7
SQP_SQUARED_TOLERANCE = 1e-10
SQP_DET_THRESHOLD = 1.001
SQP_MAX_ITERATION = 15
ORTHOGONALITY_SQUARED_ERROR_THRESHOLD = 1e-8
EQUAL_VECTORS_SQUARED_DIFF = 1e-10
EQUAL_SQUARED_ERRORS_DIFF = 1e-6
POINT_VARIANCE_THRESHOLD = 1e-5

LM_MAX_ITER = 20


# ---------------------------------------------------------------------------------------------
# small algebra
# ---------------------------------------------------------------------------------------------

def jacobi_eigh(a):
    """Eigenvalues (descending) and eigenvectors (columns) of the symmetric matrix ``a`` by cyclic
    Jacobi: a rotation whenever |a_pq| > eps sqrt(|a_pp a_qq|), until a sweep rotates nothing."""
    a = np.array(a, dtype=np.float64)
    n = a.shape[0]
    v = np.eye(n)
    for _ in range(60):
        rotated = False
        for p in range(n - 1):
            for q in range(p + 1, n):
                apq = a[p, q]
                if abs(apq) <= DBL_EPSILON * math.sqrt(abs(a[p, p] * a[q, q])) or apq == 0.0:
                    continue
                rotated = True
                theta = (a[q, q] - a[p, p]) / (2.0 * apq)
                t = 1.0 / (abs(theta) + math.sqrt(theta * theta + 1.0))
                if theta < 0:
                    t = -t
                c = 1.0 / math.sqrt(t * t + 1.0)
                s = t * c
                for k in range(n):           # columns p, q
                    akp, akq = a[k, p], a[k, q]
                    a[k, p] = c * akp - s * akq
                    a[k, q] = s * akp + c * akq
                for k in range(n):           # rows p, q
                    apk, aqk = a[p, k], a[q, k]
                    a[p, k] = c * apk - s * aqk
                    a[q, k] = s * apk + c * aqk
                for k in range(n):
                    vkp, vkq = v[k, p], v[k, q]
                    v[k, p] = c * vkp - s * vkq
                    v[k, q] = s * vkp + c * vkq
        if not rotated:
            break
    w = np.diag(a).copy()
    order = sorted(range(n), key=lambda i: -w[i])   # stable: ties keep their index order
    return w[order], v[:, order]


def svd_psd(a):
    """Singular values (descending) and left singular vectors (rows) of the symmetric positive
    semi-definite ``a``, by one-sided (Hestenes) Jacobi on its rows: each pair of rows is rotated
    until orthogonal (|a_i . a_j| <= eps |a_i| |a_j|), up to max(n, 30) sweeps, then the rows are
    sorted by norm and normalised.  EPnP's control points depend on the signs of these vectors, and
    these are the signs cv2.SVDecomp returns (to 2e-13 over random 3x3 and 12x12 inputs)."""
    at = np.array(a, dtype=np.float64)
    n = at.shape[0]
    w = np.array([at[i] @ at[i] for i in range(n)])
    for _ in range(max(n, 30)):
        changed = False
        for i in range(n - 1):
            for j in range(i + 1, n):
                p = float(at[i] @ at[j])
                if abs(p) <= DBL_EPSILON * math.sqrt(w[i] * w[j]):
                    continue
                p *= 2
                beta = w[i] - w[j]
                gamma = math.hypot(p, beta)
                if beta < 0:
                    s = math.sqrt((gamma - beta) * 0.5 / gamma)
                    c = p / (gamma * s * 2)
                else:
                    c = math.sqrt((gamma + beta) / (gamma * 2))
                    s = p / (gamma * c * 2)
                ai, aj = at[i].copy(), at[j].copy()
                at[i] = c * ai + s * aj
                at[j] = -s * ai + c * aj
                w[i], w[j] = at[i] @ at[i], at[j] @ at[j]
                changed = True
        if not changed:
            break
    sig = np.sqrt(np.einsum('ij,ij->i', at, at))
    for i in range(n - 1):   # selection sort, descending
        j = i
        for k in range(i + 1, n):
            if sig[j] < sig[k]:
                j = k
        if j != i:
            sig[[i, j]] = sig[[j, i]]
            at[[i, j]] = at[[j, i]]
    return sig, at / sig[:, None]


def cross(a, b):
    return np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


def det3(m):
    m = np.asarray(m).reshape(3, 3)
    return (m[0, 0] * (m[1, 1] * m[2, 2] - m[1, 2] * m[2, 1])
            - m[0, 1] * (m[1, 0] * m[2, 2] - m[1, 2] * m[2, 0])
            + m[0, 2] * (m[1, 0] * m[2, 1] - m[1, 1] * m[2, 0]))


def polar(a, proper=True):
    """The orthogonal factor U V^T of the 3x3 ``a`` = U S V^T, from the eigenvectors of a^T a.
    ``proper``: the nearest rotation U diag(1, 1, det(U V^T)) V^T instead."""
    a = np.asarray(a, dtype=np.float64).reshape(3, 3)
    s2, v = jacobi_eigh(a.T @ a)
    v0, v1 = v[:, 0], v[:, 1]
    u0 = a @ v0 / math.sqrt(s2[0])
    u1 = a @ v1
    u1 = u1 - (u1 @ u0) * u0
    u1 = u1 / math.sqrt(u1 @ u1)
    sign = 1.0 if proper or det3(a) >= 0 else -1.0
    return np.outer(u0, v0) + np.outer(u1, v1) + sign * np.outer(cross(u0, u1), cross(v0, v1))


def rodrigues(rvec):
    """Rotation matrix of the axis-angle vector ``rvec``."""
    r = np.asarray(rvec, dtype=np.float64).reshape(3)
    th = math.sqrt(r @ r)
    if th < DBL_EPSILON:
        return np.eye(3)
    k = r / th
    c, s = math.cos(th), math.sin(th)
    kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return c * np.eye(3) + (1 - c) * np.outer(k, k) + s * kx


def rodrigues_inv(m):
    """Axis-angle vector of the 3x3 ``m`` after projecting it on the orthogonal matrices, as
    cv2.Rodrigues does."""
    r = polar(m, proper=False)
    v = np.array([r[2, 1] - r[1, 2], r[0, 2] - r[2, 0], r[1, 0] - r[0, 1]])
    s = math.sqrt(v @ v) * 0.5
    c = min(max((r[0, 0] + r[1, 1] + r[2, 2] - 1) * 0.5, -1.0), 1.0)
    th = math.acos(c)
    if s < 1e-5:
        if c > 0:
            return np.zeros(3)
        # about pi: the axis from the diagonal, signs from the off-diagonal terms
        rx = math.sqrt(max((r[0, 0] + 1) * 0.5, 0.0))
        ry = math.sqrt(max((r[1, 1] + 1) * 0.5, 0.0)) * (-1.0 if r[0, 1] < 0 else 1.0)
        rz = math.sqrt(max((r[2, 2] + 1) * 0.5, 0.0)) * (-1.0 if r[0, 2] < 0 else 1.0)
        if abs(rx) < abs(ry) and abs(rx) < abs(rz) and ((r[1, 2] > 0) != (ry * rz > 0)):
            rz = -rz
        v = np.array([rx, ry, rz])
        return v * (th / math.sqrt(v @ v))
    return v * (th / (2.0 * s))


def rotation_jacobian(rvec):
    """J_l(rvec), the left Jacobian of SO(3): d(R(rvec) X) / d rvec = -[R X]x J_l."""
    r = np.asarray(rvec, dtype=np.float64)
    th2 = r @ r
    th = math.sqrt(th2)
    if th < 1e-5:
        a, b = 0.5, 1.0 / 6.0
    else:
        a, b = (1 - math.cos(th)) / th2, (th - math.sin(th)) / (th2 * th)
    rx = np.array([[0, -r[2], r[1]], [r[2], 0, -r[0]], [-r[1], r[0], 0]])
    return np.eye(3) + a * rx + b * (rx @ rx)


def solve_lu(a, b):
    """``a`` x = ``b`` by Gaussian elimination with partial pivoting; None when a pivot is 0."""
    a = np.array(a, dtype=np.float64)
    b = np.array(b, dtype=np.float64)
    n = a.shape[0]
    for k in range(n):
        p = k + int(np.argmax(np.abs(a[k:, k])))
        if a[p, k] == 0.0:
            return None
        if p != k:
            a[[k, p]] = a[[p, k]]
            b[[k, p]] = b[[p, k]]
        for i in range(k + 1, n):
            f = a[i, k] / a[k, k]
            a[i, k:] -= f * a[k, k:]
            b[i] -= f * b[k]
    x = np.zeros(n)
    for i in range(n - 1, -1, -1):
        x[i] = (b[i] - a[i, i + 1:] @ x[i + 1:]) / a[i, i]
    return x


def lstsq_householder(a, b):
    """Least-squares solution of the m x n ``a`` x = ``b`` (m >= n, full rank) by Householder QR."""
    a = np.array(a, dtype=np.float64)
    b = np.array(b, dtype=np.float64)
    m, n = a.shape
    for k in range(n):
        nrm = math.sqrt(a[k:, k] @ a[k:, k])
        if nrm == 0.0:
            continue
        alpha = -nrm if a[k, k] >= 0 else nrm
        v = a[k:, k].copy()
        v[0] -= alpha
        vv = v @ v
        if vv == 0.0:
            continue
        for j in range(k, n):
            a[k:, j] -= (2.0 * (v @ a[k:, j]) / vv) * v
        b[k:] -= (2.0 * (v @ b[k:]) / vv) * v
    x = np.zeros(n)
    for i in range(n - 1, -1, -1):
        x[i] = (b[i] - a[i, i + 1:n] @ x[i + 1:]) / a[i, i]
    return x


# ---------------------------------------------------------------------------------------------
# per-point terms
# ---------------------------------------------------------------------------------------------

def project(pts, rmat, t, focal):
    pc = pts @ rmat.T + t
    return focal * pc[:, :2] / pc[:, 2:3], pc


def rms_error(pts, scr, rmat, t, focal):
    """sqrt(sum |proj - screen|^2 / (2N)), the error cv2.solvePnPGeneric reports."""
    proj, _ = project(pts, rmat, t, focal)
    d = proj - scr
    return math.sqrt(float(np.sum(d * d)) / (2 * len(pts)))


# ---------------------------------------------------------------------------------------------
# SQPnP
# ---------------------------------------------------------------------------------------------

def _sqp_step(omega, r):
    """One SQP step from r (rows of R): min (r+d)^T Omega (r+d) s.t. the linearised row
    orthonormality, as its 15x15 KKT system."""
    r1, r2, r3 = r[0:3], r[3:6], r[6:9]
    jac = np.zeros((6, 9))
    jac[0, 0:3] = 2 * r1
    jac[1, 3:6] = 2 * r2
    jac[2, 6:9] = 2 * r3
    jac[3, 0:3], jac[3, 3:6] = r2, r1
    jac[4, 3:6], jac[4, 6:9] = r3, r2
    jac[5, 0:3], jac[5, 6:9] = r3, r1
    g = np.array([1 - r1 @ r1, 1 - r2 @ r2, 1 - r3 @ r3, -(r1 @ r2), -(r2 @ r3), -(r1 @ r3)])
    kkt = np.zeros((15, 15))
    kkt[:9, :9] = omega
    kkt[:9, 9:] = jac.T
    kkt[9:, :9] = jac
    rhs = np.concatenate([-(omega @ r), g])
    x = solve_lu(kkt, rhs)
    return None if x is None else x[:9]


def _run_sqp(omega, r0):
    r = r0.copy()
    for _ in range(SQP_MAX_ITERATION):
        d = _sqp_step(omega, r)
        if d is None:
            break
        r = r + d
        if d @ d <= SQP_SQUARED_TOLERANCE:
            break
    dr = det3(r)
    if dr < 0:
        r, dr = -r, -dr
    return polar(r).reshape(9) if dr > SQP_DET_THRESHOLD else r


def sqpnp(pts, scr, focal):
    """SQPnP on the normalised points scr / focal; a list of (r_hat 9, t 3) or None on failure
    (too little spread of the image points)."""
    n = len(pts)
    xy = scr / focal
    x, y = xy[:, 0], xy[:, 1]
    sq = x * x + y * y
    XX = np.einsum('ni,nj->nij', pts, pts)
    S0, Sx, Sy, Ss = (np.einsum('n,nij->ij', w, XX) for w in (np.ones(n), x, y, sq))
    sX, sxX, syX, ssX = (np.einsum('n,ni->i', w, pts) for w in (np.ones(n), x, y, sq))
    sx, sy, ss = x.sum(), y.sum(), sq.sum()
    omega = np.zeros((9, 9))
    omega[0:3, 0:3] = S0
    omega[3:6, 3:6] = S0
    omega[0:3, 6:9] = -Sx
    omega[3:6, 6:9] = -Sy
    omega[6:9, 0:3] = -Sx
    omega[6:9, 3:6] = -Sy
    omega[6:9, 6:9] = Ss
    qa = np.zeros((3, 9))    # sum_i Q_i B_i
    qa[0, 0:3], qa[0, 6:9] = sX, -sxX
    qa[1, 3:6], qa[1, 6:9] = sX, -syX
    qa[2, 0:3], qa[2, 3:6], qa[2, 6:9] = -sxX, -syX, ssX
    q = np.array([[n, 0, -sx], [0, n, -sy], [-sx, -sy, ss]], dtype=np.float64)
    detq = n * (n * ss - sy * sy - sx * sx)
    if detq / (float(n) ** 3) < POINT_VARIANCE_THRESHOLD:
        return None
    qinv = np.array([[q[1, 1] * q[2, 2] - q[1, 2] * q[2, 1], q[0, 2] * q[2, 1] - q[0, 1] * q[2, 2],
                      q[0, 1] * q[1, 2] - q[0, 2] * q[1, 1]],
                     [q[1, 2] * q[2, 0] - q[1, 0] * q[2, 2], q[0, 0] * q[2, 2] - q[0, 2] * q[2, 0],
                      q[0, 2] * q[1, 0] - q[0, 0] * q[1, 2]],
                     [q[1, 0] * q[2, 1] - q[1, 1] * q[2, 0], q[0, 1] * q[2, 0] - q[0, 0] * q[2, 1],
                      q[0, 0] * q[1, 1] - q[0, 1] * q[1, 0]]]) / detq
    pmat = -qinv @ qa
    omega = omega + qa.T @ pmat
    s, u = jacobi_eigh(omega)
    mean = sX / n
    nnull = 0
    while nnull < 8 and s[7 - nnull] < RANK_TOLERANCE:
        nnull += 1
    neig = max(nnull, 1)

    sols = []          # [r_hat, t, sq_error]
    min_err = [np.inf]

    def depth_ok(r, t):
        if r[6] * mean[0] + r[7] * mean[1] + r[8] * mean[2] + t[2] > 0:
            return True
        z = pts @ r[6:9] + t[2]
        npos = int(np.sum(z > 0))
        return npos >= n - npos

    def check(r):
        t = pmat @ r
        if not depth_ok(r, t):
            return
        err = float(r @ omega @ r)
        if abs(min_err[0] - err) > EQUAL_SQUARED_ERRORS_DIFF:
            if min_err[0] > err:
                min_err[0] = err
                sols[:] = [[r, t, err]]
        else:
            for sol in sols:
                d = sol[0] - r
                if d @ d < EQUAL_VECTORS_SQUARED_DIFF:
                    if sol[2] > err:
                        sol[:] = [r, t, err]
                    break
            else:
                if len(sols) < MAX_SQPNP_SOLUTIONS:
                    sols.append([r, t, err])
            if min_err[0] > err:
                min_err[0] = err

    def both_signs(e):
        check(_run_sqp(omega, polar(e).reshape(9)))
        check(_run_sqp(omega, polar(-e).reshape(9)))

    for i in range(9 - neig, 9):
        e = math.sqrt(3.0) * u[:, i]
        ee = e.reshape(3, 3) @ e.reshape(3, 3).T - np.eye(3)
        if float(np.sum(ee * ee)) < ORTHOGONALITY_SQUARED_ERROR_THRESHOLD:
            check(det3(e) * e)
        else:
            both_signs(e)
    c = 1
    while 9 - neig - c > 0 and min_err[0] > 3 * s[9 - neig - c]:
        both_signs(u[:, 9 - neig - c])
        c += 1
    return [(sol[0], sol[1]) for sol in sols]


# ---------------------------------------------------------------------------------------------
# EPnP
# ---------------------------------------------------------------------------------------------

_PAIRS = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))


def _epnp_pose(pts, alphas, ccs):
    pcs = alphas @ ccs
    if pcs[0, 2] < 0:
        ccs, pcs = -ccs, -pcs
    pc0, pw0 = pcs.mean(0), pts.mean(0)
    abt = (pcs - pc0).T @ (pts - pw0)
    r = polar(abt, proper=False)
    if det3(r) < 0:
        r[2] = -r[2]
    return r, pc0 - r @ pw0


def _epnp_error(pts, scr, r, t, focal):
    proj, _ = project(pts, r, t, focal)
    d = proj - scr
    return float(np.sum(np.sqrt(np.sum(d * d, 1)))) / len(pts)


def _gauss_newton(lmat, rho, betas):
    for _ in range(5):
        b0, b1, b2, b3 = betas
        a = np.stack([2 * lmat[:, 0] * b0 + lmat[:, 1] * b1 + lmat[:, 3] * b2 + lmat[:, 6] * b3,
                      lmat[:, 1] * b0 + 2 * lmat[:, 2] * b1 + lmat[:, 4] * b2 + lmat[:, 7] * b3,
                      lmat[:, 3] * b0 + lmat[:, 4] * b1 + 2 * lmat[:, 5] * b2 + lmat[:, 8] * b3,
                      lmat[:, 6] * b0 + lmat[:, 7] * b1 + lmat[:, 8] * b2 + 2 * lmat[:, 9] * b3], 1)
        prod = np.array([b0 * b0, b0 * b1, b1 * b1, b0 * b2, b1 * b2, b2 * b2, b0 * b3, b1 * b3,
                         b2 * b3, b3 * b3])
        betas = betas + lstsq_householder(a, rho - lmat @ prod)
    return betas


def epnp(pts, scr, focal):
    """EPnP; (R 3x3, t 3)."""
    n = len(pts)
    c0 = pts.mean(0)
    d = pts - c0
    w, axes = svd_psd(d.T @ d)
    cws = np.stack([c0] + [c0 + math.sqrt(w[i] / n) * axes[i] for i in range(3)])
    cc = (cws[1:] - c0).T
    alphas = np.zeros((n, 4))
    alphas[:, 1:] = d @ _inv3(cc).T
    alphas[:, 0] = 1 - alphas[:, 1:].sum(1)
    u, v = scr[:, 0], scr[:, 1]
    m = np.zeros((2 * n, 12))
    for j in range(4):
        m[0::2, 3 * j] = alphas[:, j] * focal
        m[0::2, 3 * j + 2] = -alphas[:, j] * u
        m[1::2, 3 * j + 1] = alphas[:, j] * focal
        m[1::2, 3 * j + 2] = -alphas[:, j] * v
    _, vec = svd_psd(m.T @ m)
    nv = [vec[11 - k] for k in range(4)]
    lmat = np.zeros((6, 10))
    rho = np.zeros(6)
    for i, (a, b) in enumerate(_PAIRS):
        dv = [x[3 * a:3 * a + 3] - x[3 * b:3 * b + 3] for x in nv]
        lmat[i] = [dv[0] @ dv[0], 2 * dv[0] @ dv[1], dv[1] @ dv[1], 2 * dv[0] @ dv[2],
                   2 * dv[1] @ dv[2], dv[2] @ dv[2], 2 * dv[0] @ dv[3], 2 * dv[1] @ dv[3],
                   2 * dv[2] @ dv[3], dv[3] @ dv[3]]
        e = cws[a] - cws[b]
        rho[i] = e @ e
    cand = []
    # approximation 1: [B11 B12 B13 B14]
    b4 = lstsq_householder(lmat[:, [0, 1, 3, 6]], rho)
    b = np.zeros(4)
    b[0] = math.sqrt(abs(b4[0]))
    b[1:] = (-b4[1:] if b4[0] < 0 else b4[1:]) / b[0]
    cand.append(b)
    # approximation 2: [B11 B12 B22]
    b3 = lstsq_householder(lmat[:, 0:3], rho)
    b = np.zeros(4)
    if b3[0] < 0:
        b[0] = math.sqrt(-b3[0])
        b[1] = math.sqrt(-b3[2]) if b3[2] < 0 else 0.0
    else:
        b[0] = math.sqrt(b3[0])
        b[1] = math.sqrt(b3[2]) if b3[2] > 0 else 0.0
    if b3[1] < 0:
        b[0] = -b[0]
    cand.append(b)
    # approximation 3: [B11 B12 B22 B13 B23]
    b5 = lstsq_householder(lmat[:, 0:5], rho)
    b = np.zeros(4)
    if b5[0] < 0:
        b[0] = math.sqrt(-b5[0])
        b[1] = math.sqrt(-b5[2]) if b5[2] < 0 else 0.0
    else:
        b[0] = math.sqrt(b5[0])
        b[1] = math.sqrt(b5[2]) if b5[2] > 0 else 0.0
    if b5[1] < 0:
        b[0] = -b[0]
    b[2] = b5[3] / b[0]
    cand.append(b)
    best = None
    for b in cand:
        b = _gauss_newton(lmat, rho, b)
        ccs = sum(b[k] * nv[k] for k in range(4)).reshape(4, 3)
        r, t = _epnp_pose(pts, alphas, ccs)
        err = _epnp_error(pts, scr, r, t, focal)
        if best is None or err < best[2]:
            best = (r, t, err)
    return best[0], best[1]


def _inv3(m):
    a = np.asarray(m, dtype=np.float64)
    adj = np.array([[a[1, 1] * a[2, 2] - a[1, 2] * a[2, 1], a[0, 2] * a[2, 1] - a[0, 1] * a[2, 2],
                     a[0, 1] * a[1, 2] - a[0, 2] * a[1, 1]],
                    [a[1, 2] * a[2, 0] - a[1, 0] * a[2, 2], a[0, 0] * a[2, 2] - a[0, 2] * a[2, 0],
                     a[0, 2] * a[1, 0] - a[0, 0] * a[1, 2]],
                    [a[1, 0] * a[2, 1] - a[1, 1] * a[2, 0], a[0, 1] * a[2, 0] - a[0, 0] * a[2, 1],
                     a[0, 0] * a[1, 1] - a[0, 1] * a[1, 0]]])
    return adj / det3(a)


# ---------------------------------------------------------------------------------------------
# Levenberg-Marquardt
# ---------------------------------------------------------------------------------------------

def _residuals(pts, scr, p, focal, with_jacobian):
    rmat = rodrigues(p[:3])
    proj, pc = project(pts, rmat, p[3:], focal)
    res = (proj - scr).reshape(-1)
    if not with_jacobian:
        return res, None
    n = len(pts)
    jac = np.zeros((2 * n, 6))
    iz = 1.0 / pc[:, 2]
    # d proj / d pc
    dp = np.zeros((n, 2, 3))
    dp[:, 0, 0] = focal * iz
    dp[:, 1, 1] = focal * iz
    dp[:, 0, 2] = -focal * pc[:, 0] * iz * iz
    dp[:, 1, 2] = -focal * pc[:, 1] * iz * iz
    jl = rotation_jacobian(p[:3])
    pw = pc - p[3:]
    # column k of d pc / d rvec: jl[:, k] x (R X)
    drot = np.cross(jl.T[None, :, :], pw[:, None, :]).transpose(0, 2, 1)
    jac.reshape(n, 2, 6)[:, :, :3] = dp @ drot
    jac.reshape(n, 2, 6)[:, :, 3:] = dp
    return res, jac


def refine_lm(pts, scr, rvec, t, focal):
    """(rvec, t) after OpenCV's iterative LM from the given start."""
    p = np.concatenate([np.asarray(rvec, np.float64), np.asarray(t, np.float64)])
    lam = -3
    res, jac = _residuals(pts, scr, p, focal, True)
    prev_err = math.sqrt(res @ res)
    for it in range(LM_MAX_ITER):
        jtj = jac.T @ jac
        jtr = jac.T @ res
        prev = p

        def step():
            a = jtj.copy()
            a[np.diag_indices(6)] *= 1.0 + 10.0 ** lam
            x = solve_lu(a, jtr)
            return prev - (x if x is not None else 0.0)

        p = step()
        res, _ = _residuals(pts, scr, p, focal, False)
        err = math.sqrt(res @ res)
        while err > prev_err:
            lam += 1
            if lam > 16:
                break
            p = step()
            res, _ = _residuals(pts, scr, p, focal, False)
            err = math.sqrt(res @ res)
        lam = max(lam - 1, -16)
        dp = p - prev
        if it + 1 >= LM_MAX_ITER or math.sqrt(dp @ dp) < FLT_EPSILON * math.sqrt(prev @ prev):
            break
        prev_err = err
        res, jac = _residuals(pts, scr, p, focal, True)
    return p[:3], p[3:]


# ---------------------------------------------------------------------------------------------
# the reference's function
# ---------------------------------------------------------------------------------------------

def foreground(coords, mask):
    """(points [N,3] float64, screen [N,2]) of one image, in row-major pixel order."""
    h, w = mask.shape
    idx = np.nonzero(np.asarray(mask).reshape(-1))[0]
    pts = np.asarray(coords, dtype=np.float64).reshape(-1, 3)[idx]
    scr = np.stack([(idx % w) / w, (idx // w) / h], 1) - 0.5
    return pts, scr


def solve_candidate(pts, scr, focal, refine):
    """One (image, focal) pair: a dict with solver, accepted, rvec, t, error (None when no pose)."""
    solver, rvec, t, err = SOLVER_NONE, None, None, None
    sols = sqpnp(pts, scr, focal)
    if sols:
        for r_hat, tt in sols:
            rv = rodrigues_inv(r_hat.reshape(3, 3))
            e = rms_error(pts, scr, rodrigues(rv), tt, focal)
            if tt[2] > 0 and (err is None or e < err):
                solver, rvec, t, err = SOLVER_SQPNP, rv, tt, e
    if solver == SOLVER_NONE:
        r, tt = epnp(pts, scr, focal)
        rv = rodrigues_inv(r)
        e = rms_error(pts, scr, rodrigues(rv), tt, focal)
        if tt[2] > 0:
            solver, rvec, t, err = SOLVER_EPNP, rv, tt, e
    accepted = False
    if solver != SOLVER_NONE and refine:
        rv, tt = refine_lm(pts, scr, rvec, t, focal)
        if tt[2] > 0:
            accepted = True
            rvec, t = rv, tt
            err = rms_error(pts, scr, rodrigues(rv), tt, focal)
    return dict(solver=solver, accepted=accepted, rvec=rvec, t=t, error=err)


FLIP = np.diag([1.0, -1.0, -1.0, 1.0])


def compute_pose_pnp(coords, masks, focal_proposals, refine=True, records=None):
    """The reference's compute_pose_pnp on numpy arrays: (world2cam [B,4,4], focal [B], error [B]).
    ``records``, a list, receives each image's per-candidate dicts."""
    coords = np.asarray(coords)
    masks = np.asarray(masks)
    mats, focals, errors = [], [], []
    for b in range(coords.shape[0]):
        pts, scr = foreground(coords[b], masks[b])
        best = None
        recs = []
        for focal in focal_proposals:
            if len(pts) < 4:
                break
            c = solve_candidate(pts, scr, float(focal), refine)
            recs.append(c)
            if c['solver'] != SOLVER_NONE and (best is None or c['error'] < best[0]['error']):
                best = (c, float(focal))
        if records is not None:
            records.append(recs)
        if best is None:
            rvec, t, focal, err = np.zeros(3), np.array([0.0, 0.0, -10.0]), 1.0, 10.0
        else:
            rvec, t, focal, err = best[0]['rvec'], best[0]['t'], best[1], best[0]['error']
        m = np.eye(4)
        m[:3, :3] = rodrigues(rvec)
        m[:3, 3] = t
        mats.append(FLIP @ m)
        focals.append(focal)
        errors.append(err)
    return np.stack(mats), np.array(focals, dtype=np.float64), np.array(errors, dtype=np.float64)
