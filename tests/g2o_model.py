"""CPU restatement of the reference's g2o backend (src/internal/icp-g2o.cpp) in numpy fp64, the checker of the g2o parity
tests.  Items marked [ext] are g2o's behaviour at the tag the reference's README recommends (20170730_git, README.md:65),
restated from knowledge of g2o rather than from its source (DESIGN section 2): Edge_V_V_GICP's error and analytic Jacobians,
EdgeGICP::makeRot0 / prec0, VertexSE3::oplusImpl, OptimizationAlgorithmLevenberg::solve with LinearSolverDense."""
import numpy as np

I3 = np.eye(3)


def prec0(n, eps):
    """EdgeGICP::prec0(eps) for every row of n [ext]: R0 row 2 = normal0 (not normalised), row 1 = normalise((0,1,0) - n_y n),
    row 0 = n x row 1; Omega = R0^T diag(eps, eps, 1) R0 -- not eps I + (1 - eps) n n^T, which differs for non-unit normals."""
    n = np.asarray(n, np.float64).reshape(-1, 3)
    y = np.array([0.0, 1.0, 0.0]) - n[:, 1:2] * n
    nn = np.einsum("ij,ij->i", y, y)
    y = y / np.where(nn > 0, np.sqrt(nn), 1.0)[:, None]
    R0 = np.stack([np.cross(n, y), y, n], axis=1)
    return np.einsum("nka,k,nkb->nab", R0, np.array([eps, eps, 1.0]), R0)


def skew(v):
    v = np.asarray(v).reshape(-1, 3)
    z = np.zeros(len(v))
    return np.stack([np.stack([z, -v[:, 2], v[:, 1]], 1), np.stack([v[:, 2], z, -v[:, 0]], 1),
                     np.stack([-v[:, 1], v[:, 0], z], 1)], 1)


def error(T0, T1, pos0, pos1):
    """Edge_V_V_GICP::computeError [ext]: T0^-1 (T1 pos1) - pos0 with Eigen's isometry inverse [F0^T | -F0^T t0]."""
    F0, t0, F1, t1 = T0[:3, :3], T0[:3, 3], T1[:3, :3], T1[:3, 3]
    y = pos1 @ F1.T + t1
    return y @ F0 - F0.T @ t0 - pos0


def jacobians(T0, T1, pos1):
    """GICP_ANALYTIC_JACOBIANS [ext], increment order (tx ty tz qx qy qz): J_dst = [-I | 2[u]x], J_src = [M01 | -2 M01 [pos1]x]."""
    F0, t0, F1, t1 = T0[:3, :3], T0[:3, 3], T1[:3, :3], T1[:3, 3]
    u = (pos1 @ F1.T + t1) @ F0 - F0.T @ t0
    M01 = F0.T @ F1
    N = len(pos1)
    Jd = np.concatenate([np.broadcast_to(-I3, (N, 3, 3)), 2.0 * skew(u)], axis=2)
    Js = np.concatenate([np.broadcast_to(M01, (N, 3, 3)), -2.0 * np.einsum("ij,njk->nik", M01, skew(pos1))], axis=2)
    return Jd, Js


def increment(d):
    """internal::fromVectorMQT [ext]: [R(q) | t], qw = sqrt(1 - |q|^2), the identity rotation when |q|^2 > 1."""
    qx, qy, qz = d[3:]
    w2 = 1.0 - (qx * qx + qy * qy + qz * qz)
    T = np.eye(4); T[:3, 3] = d[:3]
    if not w2 < 0:
        qw = np.sqrt(w2)
        tx, ty, tz = 2 * qx, 2 * qy, 2 * qz
        T[:3, :3] = [[1 - (ty * qy + tz * qz), ty * qx - tz * qw, tz * qx + ty * qw],
                     [ty * qx + tz * qw, 1 - (tx * qx + tz * qz), tz * qy - tx * qw],
                     [tz * qx - ty * qw, tz * qy + tx * qw, 1 - (tx * qx + ty * qy)]]
    return T


def oplus(T, d, count, ortho_after):
    """VertexSE3::oplusImpl [ext]: T <- T inc; after more than ortho_after updates F <- F - F (F^T F - I) / 2, count restarts."""
    out = np.eye(4)
    inc = increment(d)
    out[:3, :3] = T[:3, :3] @ inc[:3, :3]; out[:3, 3] = T[:3, :3] @ inc[:3, 3] + T[:3, 3]
    count += 1
    if count > ortho_after:
        count = 0
        F = out[:3, :3]
        out[:3, :3] = F - 0.5 * F @ (F.T @ F - I3)
    return out, count


class Problem:
    """The GICP edges of icp-g2o.cpp:194-256: per correspondence (first, second) of edge src -> dst, vertex 0 = dst, vertex 1 =
    src, pos0 = dst point, pos1 = src point, information I or prec0(eps) of the dst normal.  Edges between two fixed frames are
    not active; a free frame without a correspondence is not a vertex of the problem."""

    def __init__(self, pts, nor, edges, corr, fixed, point_to_plane, eps=0.01):
        self.M = len(pts)
        self.groups = []
        for (s, d), (f, sec) in zip(edges, corr):
            f = np.asarray(f, np.int64); sec = np.asarray(sec, np.int64)
            if len(f) == 0 or (fixed[s] and fixed[d]):
                continue
            Om = prec0(nor[d][sec], eps) if point_to_plane else np.broadcast_to(I3, (len(f), 3, 3))
            self.groups.append((s, d, pts[d][sec], pts[s][f], Om))
        touched = set()
        for s, d, *_ in self.groups:
            touched.update((s, d))
        self.active = [f for f in range(self.M) if f in touched and not fixed[f]]
        self.col = {f: 6 * i for i, f in enumerate(self.active)}
        self.n = 6 * len(self.active)

    def chi2(self, X):
        chi = 0.0
        for s, d, p0, p1, Om in self.groups:
            r = error(X[d], X[s], p0, p1)
            chi += float(np.einsum("ni,nij,nj->", r, Om, r))
        return chi

    def build(self, X):
        """H = sum J^T Omega J, b = -sum J^T Omega e over the free vertices, and chi2."""
        H = np.zeros((self.n, self.n)); b = np.zeros(self.n); chi = 0.0
        for s, d, p0, p1, Om in self.groups:
            r = error(X[d], X[s], p0, p1)
            chi += float(np.einsum("ni,nij,nj->", r, Om, r))
            Jd, Js = jacobians(X[d], X[s], p1)
            blocks = [(v, J) for v, J in ((d, Jd), (s, Js)) if v in self.col]
            for va, Ja in blocks:
                WJa = np.einsum("nij,njk->nik", Om, Ja)
                b[self.col[va]:self.col[va] + 6] -= np.einsum("nik,ni->k", WJa, r)
                for vb, Jb in blocks:
                    H[self.col[vb]:self.col[vb] + 6, self.col[va]:self.col[va] + 6] += np.einsum("nib,nia->ba", Jb, WJa)
        return H, b, chi


def _solve_dense(A, b):
    """LinearSolverDense [ext]: a dense LDL^T of the (symmetric) system; None when it is not positive definite."""
    n = len(b)
    L = np.eye(n); D = np.zeros(n)
    for j in range(n):
        D[j] = A[j, j] - (L[j, :j] ** 2) @ D[:j]
        if not D[j] > 0:
            return None
        L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ (D[:j] * L[j, :j])) / D[j]
    z = np.linalg.solve(L, b)
    return np.linalg.solve(L.T, z / D)


def optimize(problem, poses, iterations=100, max_calls=100, no_improvement_limit=5, max_trials=10, tau=1e-5,
             ortho_after=1000):
    """OptimizationAlgorithmLevenberg::solve inside SparseOptimizer::optimize(iterations) [ext], called as the reference's
    outer loop does (icp-g2o.cpp:261-303; the pairwise solvers: one call, iterations = 300, max_calls = 1).
    Returns (poses, summary dict, chi2 before the first call and after each call, trial trace rows (lambda, chi, tchi, rho,
    accepted))."""
    X = [np.array(P, np.float64) for P in poses]
    count = {f: 0 for f in problem.active}
    trace = []
    summ = dict(calls=0, iterations=0, trials=0, accepted=0)
    if problem.n == 0:
        return np.stack(X), dict(summ, ended=2), np.zeros(0), np.zeros((0, 5))
    chi_init = problem.chi2(X)
    chis = [chi_init]; last = chi_init; no_impr = 0; ended = 1
    lam = nu = 0.0
    for call in range(max_calls):
        for it in range(iterations):
            H, b, chi = problem.build(X)
            if it == 0:
                lam = tau * float(np.max(np.abs(np.diag(H)))); nu = 2.0
            q = 0
            while True:
                dx = _solve_dense(H + lam * np.eye(problem.n), b)
                Xt = list(X)
                for f in problem.active:   # the update is applied (and counted) even when the factorisation failed
                    c = problem.col[f]
                    Xt[f], count[f] = oplus(X[f], dx[c:c + 6] if dx is not None else np.zeros(6), count[f], ortho_after)
                if dx is not None:
                    tchi = problem.chi2(Xt)
                    rho = (chi - tchi) / (float(dx @ (lam * dx + b)) + 1e-3)
                else:
                    tchi, rho = np.inf, -np.inf
                acc = rho > 0 and np.isfinite(tchi)
                trace.append((lam, chi, tchi, rho, float(acc)))
                if acc:
                    lam *= max(1.0 / 3.0, min(2.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3)); nu = 2.0; chi = tchi; X = Xt
                    summ["accepted"] += 1
                else:
                    lam *= nu; nu *= 2.0
                q += 1; summ["trials"] += 1
                if not (rho < 0 and q < max_trials):
                    break
            summ["iterations"] += 1
            if q == max_trials or rho == 0:
                break
        new = problem.chi2(X)
        chis.append(new)
        impr = (last - new) / last if last != 0 else np.nan
        last = new
        summ["calls"] += 1
        if not impr > 0:
            no_impr += 1
        if no_impr > no_improvement_limit:
            ended = 0
            break
    out = np.stack([np.array(P, np.float64) for P in poses])
    for f in problem.active:
        out[f] = X[f]
    summ.update(ended=ended, chi2_initial=chi_init, chi2_final=chis[-1])
    return out, summ, np.array(chis), np.array(trace).reshape(-1, 5)
