"""Per-edge normal equations of the LM step (lm_eval_kernel / lm_eval_general_kernel + lm_edge_kernel / lm_edge_general_kernel)
against an extended-precision evaluation of the reference's cost functors, read edge by edge with mvicp_debug_edge_blocks.

Reference.  The functors of icp-ceres.h restated in numpy.longdouble (64-bit mantissa on x86-64), in WORLD frame and per frame
as y(v) = R v + t with, per local tangent direction j, d y / d delta_j = D_j v + c_j: the ambient derivative of the functor
times the parameterisation's plus-Jacobian at delta = 0.  Angle-axis: Ceres' Rodrigues (D_j = R [Jr e_j]x, exact Jr) or, for
theta^2 <= DBL_EPSILON, its first-order branch p + w x p (D_j = [e_j]x); the plus is addition.  Quaternion: the polynomial map
F(q) (matrix_of_quat, unit or not) and EigenQuaternionParameterization's plus [d, 0] (x) q.  SE3: F(q) and x * exp(delta)
with the renormalisation of the quaternion (the autodiff plus).  Residuals: point-to-point d = y_s(p) - y_k(q), point-to-plane
d . F_k n, both for MIXED; SoftLOneLoss(a = edge weight) scales each block's rows by sqrt(rho') (rho'' < 0).  Output per edge:
the 12x12 Gauss-Newton block [src | dst], the 12-gradient and the cost, in the parameterisation's tangent order.

Tolerance.  Not fitted: each entry must satisfy |engine - reference| <= gamma_k * magnitude, gamma_k = k u / (1 - k u),
u = 2^-53, where `magnitude` is the same evaluation in magnitude arithmetic (every input by its absolute value, every
subtraction an addition) following the engine's own formulation: the pose matrices from the parameters, R_rel / t_rel and the
dst-frame rows of lm_eval_kernel with lm_edge_kernel's expansion [I | -Q] and K_pair, or the world-frame rows of the general
frame model, and the robust weight's dependence on the squared residual.  k (see `k_depth`) is the operation depth per
correspondence plus the slots per thread, the warp and CTA reduction, the tiles of the edge and the expansion.  A dropped,
duplicated or mis-weighted correspondence moves an entry by a whole term of its sum, a wrong tangent map a whole block: both
far above this bound.  The blocks assembled over the free frames are held to the same bound against oracle.evaluate.

Two model differences are allowed for, both O(theta) and only where they arise (DESIGN section 4.3): below theta^2 =
DBL_EPSILON the engine's angle-axis Jacobian is -(I + [w]x)[p]x where Ceres' is -[p]x (a Cauchy-Schwarz allowance,
O(theta) on that frame's rows and columns and O(theta^2) elsewhere on its edges), and the oracle's Rodrigues jets lose accuracy for
0 < theta < 1: angle-axis sets with such an angle skip the oracle, one set of angles 0 and 1.5 ... pi pins it."""
import ctypes as C
import math

import numpy as np
import pytest

from mv_lm_icp_b200 import COST_MIXED, COST_P2P, COST_P2PLANE, PARAM_AA, PARAM_QUAT, PARAM_SE3, Engine
from mv_lm_icp_b200._lib import MvicpError, check
from mv_lm_icp_b200.api import TERMINATION, default_options
from test_gpu_lm_graphs import MODES, OFF_GRID, _f32_exact, _fixed_list, compare_solve, tile_len, tile_scene

pytestmark = pytest.mark.gpu
LD = np.longdouble
EOUT = 160
U = 2.0 ** -53
EPS = 2.220446049250313e-16
PARAMS = [PARAM_AA, PARAM_QUAT, PARAM_SE3]
COSTS = [COST_P2P, COST_P2PLANE, COST_MIXED]
ROBUST = {"off": None, "edge": 0.0, "tiny": 1e-6, "huge": 1e6}   # None: no loss; 0.0: the scene's weights; else every weight


# ---- the readout ---------------------------------------------------------------------------------------------------------
def edge_blocks(eng):
    """mvicp_debug_edge_blocks: [E, 160] = Hp (12x12 row-major, src then dst) | gp (12) | cost | 3 zeros."""
    lib = eng._l
    n = C.c_int32(0)
    check(lib.mvicp_debug_edge_blocks(eng._ctx, None, C.c_int64(0), C.byref(n)))
    out = np.full((n.value, EOUT), np.nan)
    check(lib.mvicp_debug_edge_blocks(eng._ctx, out.ctypes.data_as(C.POINTER(C.c_double)), C.c_int64(out.size), C.byref(n)))
    return out


# ---- extended-precision frame models -----------------------------------------------------------------------------------
def _skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]], dtype=v.dtype)


def _series(th2, first):
    """sum_k (-th2)^k / (2k + first)!  (sinc: first = 1; (1 - cos)/th^2: 2; (th - sin)/th^3: 3), to 20 terms."""
    s, term = LD(0), LD(1) / LD(math.factorial(first))
    for k in range(20):
        s += term
        term *= -th2 / LD((2 * k + first + 1) * (2 * k + first + 2))
    return s


def _trig(th2):
    th = np.sqrt(th2)
    if th < 1:
        return _series(th2, 1), _series(th2, 2), _series(th2, 3)
    return np.sin(th) / th, (1 - np.cos(th)) / th2, (th - np.sin(th)) / (th2 * th)


def _quat_prod(a, b):
    return np.array([a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1],
                     a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2],
                     a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0],
                     a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]])


class Frame:
    """y(v) = R v + t, d y / d delta_j = D[j] v + c[j] (longdouble), and the magnitudes the engine's arithmetic carries:
    Rm (|R| through its formula), Dm, cm, Km (|K| of tangent_map, unit path)."""

    def __init__(self, param, x):
        x = np.asarray(x, np.float64)
        E3 = np.eye(3, dtype=LD)
        self.D = np.zeros((6, 3, 3), LD); self.c = np.zeros((6, 3), LD)
        self.Dm = np.zeros((6, 3, 3), LD); self.cm = np.zeros((6, 3), LD)
        self.Km = np.zeros((6, 6), LD)
        if param == PARAM_AA:
            w = x[:3].astype(LD); self.t = x[3:].astype(LD)
            self.theta = float(np.sqrt(w @ w))
            W = _skew(w); Wm = np.abs(W)
            th2_engine = x[0] * x[0] + x[1] * x[1] + x[2] * x[2]       # the branch test of rotation_of_aa_functor, in fp64
            if not th2_engine > EPS:                                      # Ceres' first-order branch: p + w x p
                self.R = E3 + W; self.Rm = E3 + Wm
                for j in range(3):
                    self.D[j] = _skew(E3[j])
                Jrm = E3
                self.small = th2_engine > 0
            else:
                th2 = w @ w; th = np.sqrt(th2)
                sinc, a, b = _trig(th2)
                self.R = E3 + sinc * W + a * W @ W
                Jr = E3 - a * W + b * W @ W
                for j in range(3):
                    self.D[j] = self.R @ _skew(Jr[:, j])
                # matrix_of_aa: c I + (1 - c) k k^T + s [k]x with k = w / th: 1 - c carries |c| + 1
                cs, sn, k = abs(np.cos(th)), abs(np.sin(th)), np.abs(w) / th
                self.Rm = cs * E3 + (1 + cs) * np.outer(k, k) + sn * np.abs(_skew(k))
                # so3_right_jacobian: the series below th = 1e-4, else (1 - cos) / th^2 and (th - sin) / th^3
                a_m, b_m = (a, b) if float(th) < 1e-4 else ((1 + cs) / th2, (th + sn) / (th2 * th))
                Jrm = E3 + a_m * Wm + b_m * Wm @ Wm
                self.small = False
            for j in range(3):
                self.Dm[j] = self.Rm @ np.abs(_skew(Jrm[:, j]))
                self.c[3 + j] = E3[j]; self.cm[3 + j] = E3[j]
            self.Km[3:, :3] = Jrm; self.Km[:3, 3:] = self.Rm.T
            return
        self.small = False; self.theta = 0.0
        q = x[:4].astype(LD); self.t = x[4:].astype(LD)
        u = q[:3]; w = q[3]
        Uq = _skew(u); Um = np.abs(Uq)
        self.R = E3 + 2 * w * Uq + 2 * Uq @ Uq
        self.Rm = E3 + 2 * abs(w) * Um + 2 * Um @ Um
        dF = [2 * w * _skew(E3[c]) + 2 * (_skew(E3[c]) @ Uq + Uq @ _skew(E3[c])) for c in range(3)] + [2 * Uq]
        dFm = [2 * abs(w) * np.abs(_skew(E3[c])) + 2 * (np.abs(_skew(E3[c])) @ Um + Um @ np.abs(_skew(E3[c]))) for c in range(3)] + [2 * Um]
        P = np.zeros((4, 6), LD); Pm = np.zeros((4, 6), LD)
        if param == PARAM_QUAT:       # [d, 0] (x) q; t additive; tangent (dq, dt)
            for j in range(3):
                e = np.zeros(4, LD); e[j] = 1
                P[:, j] = _quat_prod(e, q); Pm[:, j] = np.abs(P[:, j])
                self.c[3 + j] = E3[j]; self.cm[3 + j] = E3[j]
            self.Km[3:, :3] = 2 * self.Rm.T; self.Km[:3, 3:] = self.Rm.T
        else:                         # normalise(q (x) [omega / 2, 1]); t + F(q) upsilon; tangent (upsilon, omega)
            n2 = q @ q; nn = np.sqrt(n2)
            for i in range(3):
                h = np.zeros(4, LD); h[i] = LD(0.5)
                g = _quat_prod(q, h)
                P[:, 3 + i] = (g - q * (g @ q) / n2) / nn
                Pm[:, 3 + i] = (np.abs(g) + np.abs(q) * (np.abs(g) @ np.abs(q)) / n2) / nn
                self.c[i] = self.R[:, i]; self.cm[i] = self.Rm[:, i]
            self.Km = np.eye(6, dtype=LD)
        for j in range(6):
            self.D[j] = sum(P[c, j] * dF[c] for c in range(4))
            self.Dm[j] = sum(Pm[c, j] * dFm[c] for c in range(4))


# ---- parameters the engine derives from a pose (param_of_pose), restated in fp64 ---------------------------------------
def quat_of_matrix(m):
    m = m.ravel()
    tr = m[0] + m[4] + m[8]
    q = np.zeros(4)
    if tr > 0.0:
        s = math.sqrt(tr + 1.0); q[3] = 0.5 * s; s = 0.5 / s
        q[0] = (m[7] - m[5]) * s; q[1] = (m[2] - m[6]) * s; q[2] = (m[3] - m[1]) * s
    else:
        i = 0
        if m[4] > m[0]: i = 1
        if m[8] > m[4 * i]: i = 2
        j = (i + 1) % 3; k = (j + 1) % 3
        s = math.sqrt(m[4 * i] - m[4 * j] - m[4 * k] + 1.0)
        q[i] = 0.5 * s; s = 0.5 / s
        q[3] = (m[3 * k + j] - m[3 * j + k]) * s
        q[j] = (m[3 * j + i] + m[3 * i + j]) * s
        q[k] = (m[3 * k + i] + m[3 * i + k]) * s
    return q


def quat_branch(m):
    """-1: positive-trace branch of quat_of_matrix, else the index i of the largest diagonal."""
    m = m.ravel()
    if m[0] + m[4] + m[8] > 0.0:
        return -1
    i = 0
    if m[4] > m[0]: i = 1
    if m[8] > m[4 * i]: i = 2
    return i


def aa_of_matrix(m):
    mm = m.ravel()
    tr = mm[0] + mm[4] + mm[8]
    if tr >= 0.0:                     # unlike quat_of_matrix, the positive branch includes trace 0
        s = math.sqrt(tr + 1.0); w = 0.5 * s; s = 0.5 / s
        x, y, z = (mm[7] - mm[5]) * s, (mm[2] - mm[6]) * s, (mm[3] - mm[1]) * s
    else:
        x, y, z, w = quat_of_matrix(m)
    s2 = x * x + y * y + z * z
    if s2 > 0.0:
        sn = math.sqrt(s2)
        two_theta = 2.0 * (math.atan2(-sn, -w) if w < 0.0 else math.atan2(sn, w))
        kk = two_theta / sn
        return np.array([x * kk, y * kk, z * kk])
    return np.array([x * 2.0, y * 2.0, z * 2.0])


def param_of_pose(param, P):
    R, t = P[:3, :3], P[:3, 3]
    return np.concatenate([aa_of_matrix(R) if param == PARAM_AA else quat_of_matrix(R), t])


# ---- reference blocks and their magnitudes ---------------------------------------------------------------------------
def _cross_m(a, b):
    return np.stack([a[:, 1] * b[:, 2] + a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] + a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] + a[:, 1] * b[:, 0]], 1)


def _skew_m(v):
    """|[v]x| for a batch [n, 3] -> [n, 3, 3]."""
    z = np.zeros(len(v), LD)
    return np.stack([np.stack([z, v[:, 2], v[:, 1]], 1), np.stack([v[:, 2], z, v[:, 0]], 1), np.stack([v[:, 1], v[:, 0], z], 1)], 1)


def _loss(s, s_m, b):
    """(weight sqrt(rho')^2 = rho', cost, |weight|, |cost|) per residual block; b None: no loss."""
    if b is None:
        one = np.ones_like(s)
        return one, s / 2, one, s_m / 2
    w = 1 / np.sqrt(1 + s / b)
    cost = s / (np.sqrt(1 + s / b) + 1)                 # b (sqrt(1 + s/b) - 1) without the cancellation
    return w, cost, w + w ** 3 * s_m / (2 * b), b * np.sqrt(1 + s_m / b) + w * s_m / 2


def reference_edge(Fs, Fk, p, q, n, cost, b, general):
    """(H 12x12, g 12, cost) of one edge in longdouble and their magnitudes (H_m, g_m, cost_m) in the engine's formulation:
    the general frame model's world-frame rows, or the unit path's dst-frame rows expanded through [I | -Q] and K_pair."""
    p = p.astype(LD); q = q.astype(LD)
    ap, aq = np.abs(p), np.abs(q)
    H = np.zeros((12, 12), LD); g = np.zeros(12, LD); c = LD(0)
    Hm = np.zeros((12, 12), LD); gm = np.zeros(12, LD); cm = LD(0)
    d = (p @ Fs.R.T + Fs.t) - (q @ Fk.R.T + Fk.t)
    Js = np.stack([p @ Fs.D[j].T + Fs.c[j] for j in range(6)], 2)           # [n, 3, 6]
    Jk = -np.stack([q @ Fk.D[j].T + Fk.c[j] for j in range(6)], 2)
    J3 = np.concatenate([Js, Jk], 2)                                        # [n, 3, 12]
    # world-frame magnitudes: the general path's formulation; on the unit path they bound what its use of R^T R = I (the pose
    # matrices are orthogonal to a few u) and of the moments leaves out
    dw_m = (ap @ Fs.Rm.T + np.abs(Fs.t)) + (aq @ Fk.Rm.T + np.abs(Fk.t))
    J3m = np.concatenate([np.stack([ap @ Fs.Dm[j].T + Fs.cm[j] for j in range(6)], 2),
                          np.stack([aq @ Fk.Dm[j].T + Fk.cm[j] for j in range(6)], 2)], 2)
    if general:
        d_m = dw_m
    else:                             # lm_eval_kernel: x = R_rel p + t_rel, d = x - q in the dst frame
        Rrel_m = Fk.Rm.T @ Fs.Rm
        trel_m = Fk.Rm.T @ (np.abs(Fs.t) + np.abs(Fk.t))
        d_m = ap @ Rrel_m.T + trel_m + aq
        Q_m = np.zeros((6, 6), LD)
        Q_m[:3, :3] = Rrel_m.T; Q_m[:3, 3:] = Rrel_m.T @ np.abs(_skew(trel_m)); Q_m[3:, 3:] = Rrel_m.T
        Kp_m = np.zeros((12, 12), LD); Kp_m[:6, :6] = Fs.Km; Kp_m[6:, 6:] = Fk.Km
    blocks = []
    if cost != COST_P2PLANE:
        blocks.append("p2p")
    if cost != COST_P2P:
        blocks.append("plane")
    Hc_m = np.zeros((12, 12), LD); gc_m = np.zeros(12, LD)
    for kind in blocks:
        if kind == "p2p":
            r = d; J = J3
            s = np.sum(d * d, 1)
            s_m = np.sum(d_m * d_m, 1) + (0 if general else np.sum(dw_m * dw_m, 1))
        else:
            nn = n.astype(LD); an = np.abs(nn)
            m = nn @ Fk.R.T
            r = np.sum(d * m, 1)[:, None]
            Jd = np.stack([nn @ Fk.D[j].T for j in range(6)], 2)             # d (F_k n) / d delta_k
            J = np.einsum("ni,nij->nj", m, J3)[:, None, :]
            J[:, 0, 6:] += np.einsum("ni,nij->nj", d, Jd)
            mw_m = an @ Fk.Rm.T
            if general:
                m_m = mw_m
                s_m = np.sum(d_m * m_m, 1) ** 2
            else:
                m_m = an @ Rrel_m                                           # R_rel^T n
                s_m = np.sum(d_m * an, 1) ** 2 + np.sum(dw_m * mw_m, 1) ** 2
            s = r[:, 0] ** 2
        w, cst, w_m, cst_m = _loss(s, s_m, b)
        H += np.einsum("n,nia,nib->ab", w, J, J)
        g += np.einsum("n,nia,ni->a", w, J, r)
        c += np.sum(cst); cm += np.sum(cst_m)
        if kind == "p2p":
            Jm, rm = J3m, dw_m
        else:
            Jdm = np.stack([an @ Fk.Dm[j].T for j in range(6)], 2)
            Jm = np.einsum("ni,nij->nj", mw_m, J3m)[:, None, :]
            Jm[:, 0, 6:] += np.einsum("ni,nij->nj", dw_m, Jdm)
            rm = np.sum(dw_m * mw_m, 1)[:, None]
        Hm += np.einsum("n,nia,nib->ab", w_m, Jm, Jm)
        gm += np.einsum("n,nia,ni->a", w_m, Jm, rm)
        if not general:
            if kind == "p2p":         # canonical rows: src [I | [p]x], dst R_rel [I | [q]x] (the moments of lm_edge_kernel)
                I3 = np.broadcast_to(np.eye(3, dtype=LD), (len(p), 3, 3))
                Gs = np.concatenate([I3, _skew_m(ap)], 2)
                Gk = np.einsum("ij,njk->nik", Rrel_m, np.concatenate([I3, _skew_m(aq)], 2))
                Jc = np.concatenate([Gs, Gk], 2)
                u_m = d_m @ Rrel_m
                gsrc = np.concatenate([u_m, _cross_m(ap, u_m)], 1)
            else:                     # a = [m ; p x m], dst side a Q
                a_m = np.concatenate([m_m, _cross_m(ap, m_m)], 1)
                Jc = np.concatenate([a_m, a_m @ Q_m], 1)[:, None, :]
                gsrc = np.sum(d_m * an, 1)[:, None] * a_m
            Hc_m += np.einsum("n,nia,nib->ab", w_m, Jc, Jc)
            gs_ = np.einsum("n,na->a", w_m, gsrc)
            gc_m[:6] += gs_; gc_m[6:] += Q_m.T @ gs_
    if not general:
        Hm += Kp_m.T @ Hc_m @ Kp_m; gm += Kp_m.T @ gc_m
    return H, g, c, Hm, gm, cm


K_CORR = 40      # per correspondence: R_rel 3, t_rel 4, x 4, d 1, r 3, s 1 (p2p 5), w 3 (rsqrt 1 ulp), m 3, p x m 2, products 2,
                 # the 4 terms of the general row (D_j: 3 + 4, F 3) -- 40 bounds the longer of the two paths
K_POSE = 24      # parameters from the pose (param_of_pose: sqrt, division, atan2 <= 2 ulp, the AA scaling) 12, R / F / Jr from them 12
K_EXPAND = 30    # lm_edge_kernel: Q 4, A Q 6, Q^T A Q 6, Hcan K 6, K^T T1 6, -Q^T b 2 (the general path only re-adds partials)


def k_depth(tl, n_src):
    return K_CORR + K_POSE + K_EXPAND + tl // 256 + 13 + max(1, -(-n_src // tl))


def gamma(k):
    return k * U / (1 - k * U)


# ---- scenes ----------------------------------------------------------------------------------------------------------
def _rot(axis, th):
    a = np.asarray(axis, LD); a = a / np.sqrt(a @ a)
    sinc, aa, _ = _trig(LD(th) * LD(th)) if th else (LD(1), LD(0.5), None)
    W = _skew(a * LD(th))
    return (np.eye(3, dtype=LD) + sinc * W + aa * W @ W).astype(np.float64)


AXIS = (0.3, -0.5, 0.8)
SQ = math.sqrt(EPS)


def rotations(param):
    """The rotations of the block cases: (name, 3x3).  Angle-axis: the branch points of rotation_of_aa_functor and
    so3_right_jacobian and the neighbourhood of pi; quaternion / SE3: each branch of quat_of_matrix."""
    if param == PARAM_AA:
        rs = [("0", np.eye(3)), ("th2_below_eps", _rot(AXIS, SQ * (1 - 1e-3))), ("th2_above_eps", _rot(AXIS, SQ * (1 + 1e-3))),
              ("1e-4_below", _rot(AXIS, 1e-4 * (1 - 1e-12))), ("1e-4_above", _rot(AXIS, 1e-4 * (1 + 1e-12))), ("1", _rot(AXIS, 1.0)),
              ("pi-1e-6", _rot(AXIS, math.pi - 1e-6)), ("pi", np.diag([1.0, -1.0, -1.0]))]
    else:
        third = 2 * math.pi / 3      # trace 1 + 2 cos(theta) crosses 0 here
        rs = [("trace>0", _rot(AXIS, 0.3)), ("trace_just>0", _rot(AXIS, third - 1e-9)), ("trace_just<0", _rot(AXIS, third + 1e-9)),
              ("i0", _rot((0.9, 0.3, -0.3), math.pi - 1e-6)), ("i1", _rot((0.3, -0.9, 0.3), math.pi - 1e-6)),
              ("i2_qw~0", _rot((-0.3, 0.3, 0.9), math.pi - 1e-6)), ("i1_pi", np.diag([-1.0, 1.0, -1.0])), ("i2_pi", np.diag([-1.0, -1.0, 1.0]))]
        expect = [-1, -1, 2, 0, 1, 2, 1, 2]
        assert [quat_branch(R) for _, R in rs] == expect, [quat_branch(R) for _, R in rs]
        assert quat_of_matrix(rs[2][1])[3] > 0 and abs(rs[2][1].trace()) < 1e-8 and abs(rs[1][1].trace()) < 1e-8
    return rs


def pose_sets(param, n_frames, general, rng):
    """Pose sets that put every rotation of `rotations(param)` on some frame (frame 0 included: it is the fixed dst of several
    edges).  General: every pose scaled by 1 + 1e-3 (non-unit quaternion, same quat_of_matrix branch)."""
    rs = rotations(param)
    groups = [[rs[(i0 + f) % len(rs)] for f in range(n_frames)] for i0 in range(0, len(rs), n_frames)]
    if param == PARAM_AA:             # one set of angles 0 and >= 1 only: the set on which the oracle is pinned (compare_blocks)
        big = [("0", np.eye(3)), ("1.5", _rot(AXIS, 1.5)), ("2.5", _rot((0.8, 0.5, -0.3), 2.5)), ("pi-1e-6", _rot(AXIS, math.pi - 1e-6)),
               ("pi", np.diag([1.0, -1.0, -1.0])), ("3", _rot((-0.2, 0.9, 0.4), 3.0))]
        groups.append([big[f % len(big)] for f in range(n_frames)])
    out = []
    for grp in groups:
        P = np.stack([np.eye(4)] * n_frames)
        names = []
        for f in range(n_frames):
            name, R = grp[f]
            P[f, :3, :3] = R * (1 + 1e-3) if general else R
            P[f, :3, 3] = rng.uniform(-0.2, 0.2, 3)
            names.append(name)
        out.append((names, P))
    return out


def block_scene(tl, offset=0.0, f64=False):
    """tile_scene(tl) plus a general-path pairing edge: 3 inliers ending on the last slot of the second tile of frame 4."""
    pts, nor, poses, edges, corr, w, active = tile_scene(tl)
    T = tl
    edges = edges + [(4, 3)]
    corr = corr + [(np.array([2 * T - 3, 2 * T - 2, 2 * T - 1], np.int32), np.array([5, 0, T], np.int32))]
    w = w + [np.float32(0.3)]
    if f64:
        pts = [p + offset + OFF_GRID for p in pts]
    return pts, nor, edges, corr, w, active + len(pts[4])


# ---- the check -------------------------------------------------------------------------------------------------------
def compare_blocks(eng, O, pts, nor, poses, edges, corr, w, fixed, param, cost, b_over, tl, what, use_oracle=True):
    """One evaluation at `poses` (max_num_iterations = 0); every edge held to gamma_k * magnitude; the assembled blocks against
    oracle.evaluate.  b_over: None no loss, 0 the edges' weights, else every edge's weight.  Returns the worst error / bound."""
    robust = b_over is not None
    wts = [np.float32(x) if (b_over in (None, 0.0) or not len(corr[e][0])) else np.float32(b_over) for e, x in enumerate(w)]
    eng.set_poses(poses, fixed)
    for e in range(len(edges)):
        eng.set_edge(e, corr[e][0], corr[e][1], wts[e])
    opt = default_options(); opt.max_num_iterations = 0
    s = eng.optimize(param, cost, robust, options=opt)
    assert TERMINATION[s["termination"]] == "MAX_ITERATIONS", (what, s)
    out = edge_blocks(eng)
    general = param != PARAM_AA and any(abs(np.linalg.det(P[:3, :3]) - 1) > 1e-9 for P in poses)
    frames = [Frame(param, param_of_pose(param, P)) for P in poses]
    if not general:                   # the restated pose -> parameter step reproduces the pose (every quat_of_matrix branch)
        for f, P in enumerate(poses):
            assert np.max(np.abs(frames[f].R.astype(np.float64) - P[:3, :3])) <= 64 * U, (what, f)
    free = [f for f in range(len(poses)) if not fixed[f]]
    col = {f: 6 * i for i, f in enumerate(free)}
    n = 6 * len(free)
    Ha, ga, Ham, gam = (np.zeros((n, n), LD), np.zeros(n, LD), np.zeros((n, n), LD), np.zeros(n, LD))
    worst = 0.0
    for e, (sf, df) in enumerate(edges):
        o = out[e]
        assert np.all(np.isfinite(o)), (what, e)
        if fixed[sf] or not len(corr[e][0]):
            assert not np.any(o), (what, e, "an edge without residuals must hold exact zeros")
            continue
        first, second = corr[e]
        b = None if not robust else LD(float(wts[e])) ** 2
        H, g, c, Hm, gm, cm = reference_edge(frames[sf], frames[df], pts[sf][first], pts[df][second],
                                             None if cost == COST_P2P else nor[df][second], cost, b, general)
        gam_k = gamma(k_depth(tl, len(pts[sf])))
        got = np.concatenate([o[:144], o[144:156], o[156:157]]).astype(LD)
        ref = np.concatenate([H.ravel(), g, [c]]); mag = np.concatenate([Hm.ravel(), gm, [cm]])
        err = np.abs(got - ref); bound = gam_k * mag
        # Below theta^2 = DBL_EPSILON the engine's angle-axis rotation column is -(I + [w]x)[p]x e_a, Ceres' -[p]x e_a, and its
        # canonical formulation takes R = I + [w]x for orthogonal, which it is to theta^2: a column of that frame moves by at
        # most theta times its own length, any other by theta^2.  An entry of H then moves by at most that factor times
        # sqrt(H_aa H_bb) per moved column (Cauchy-Schwarz), a gradient entry by sqrt(H_aa sum w r^2), sum w r^2 <= 4 cost;
        # with magnitudes for the sums and a factor 2 of slack
        for f, off in ((sf, 0), (df, 6)):
            if frames[f].small:
                th = frames[f].theta
                col_f = np.full(12, th * th); col_f[off:off + 6] = th
                dH = np.sqrt(np.outer(np.diag(Hm), np.diag(Hm))) * (col_f[:, None] + col_f[None, :])
                dg = np.sqrt(np.diag(Hm) * 4 * cm) * col_f
                bound = bound + 2 * np.concatenate([dH.ravel(), dg, [0]])
        bad = np.nonzero(err > bound)[0]
        if len(bad):
            i = int(bad[np.argmax((err / np.maximum(bound, 1e-300))[bad])])
            where = f"H[{i // 12}][{i % 12}]" if i < 144 else (f"g[{i - 144}]" if i < 156 else "cost")
            raise AssertionError(f"{what} edge {e} ({sf}->{df}, {len(first)} inliers): {len(bad)} entries out of bound; worst {where}: "
                                 f"engine {float(got[i]):.17g} reference {float(ref[i]):.17g} |diff| {float(err[i]):.3g} bound {float(bound[i]):.3g}")
        worst = max(worst, float(np.max(err / np.maximum(bound, 1e-300))))
        for (fa, oa), (fb, ob) in [((sf, 0), (sf, 0)), ((sf, 0), (df, 6)), ((df, 6), (sf, 0)), ((df, 6), (df, 6))]:
            if fa in col and fb in col:
                Ha[col[fa]:col[fa] + 6, col[fb]:col[fb] + 6] += H[oa:oa + 6, ob:ob + 6]
                Ham[col[fa]:col[fa] + 6, col[fb]:col[fb] + 6] += Hm[oa:oa + 6, ob:ob + 6]
        for f, oa in ((sf, 0), (df, 6)):
            if f in col:
                ga[col[f]:col[f] + 6] += g[oa:oa + 6]; gam[col[f]:col[f] + 6] += gm[oa:oa + 6]
    # Ceres' Rodrigues jets (and the oracle's restatement of them) lose about u / theta in the angle-axis Jacobian for
    # 0 < theta < 1; the engine's right Jacobian does not (series below 1e-4), so only sets without such angles pin the oracle
    pinned = use_oracle and not (param == PARAM_AA and any(0 < fr.theta < 1 for fr in frames))
    if pinned:
        nr = [None] * len(pts) if cost == COST_P2P else nor
        _, Ho, go = O.evaluate(pts, nr, poses, edges, corr, wts, param=param, cost=cost, robust=robust, threads=8, fixed=fixed)
        kk = gamma(k_depth(tl, max(len(p) for p in pts)) + len(edges))
        for name, got, ref, mag in (("H", Ho, Ha, Ham), ("g", go, ga, gam)):
            err = np.abs(got.astype(LD) - ref)
            r_ = err / np.maximum(kk * mag, 1e-300)
            i_ = np.unravel_index(int(np.argmax(r_)), r_.shape)
            assert np.all(err <= kk * mag), (what, "oracle", name, i_, float(r_[i_]), float(got[i_]), float(ref[i_]), float(mag[i_]))
    return worst, pinned


def run_block_cases(O, tl, mode, params=PARAMS, costs=COSTS, robusts=tuple(ROBUST), paths=("unit", "general"), offset=0.0,
                    use_oracle=True):
    pts, nor0, edges, corr, w, active = block_scene(tl, offset, mode == "f64")
    assert tile_len(active) == tl, (active, tile_len(active))
    assert _f32_exact(np.concatenate(pts)) == (mode != "f64")
    eng = Engine(); eng.set_frames(pts, None if mode == "f32_no_normals" else nor0); eng.set_graph(edges)
    nor = nor0
    if mode == "f32_recomputed_normals":
        nor, _ = eng.recompute_normals(10)
        assert not all(_f32_exact(x) for x in nor)
    fixed = _fixed_list(len(pts), (0,))
    rng = np.random.default_rng(tl)
    worst, oracle_sets = 0.0, set()
    try:
        for path in paths:
            for param in params:
                if path == "general" and param == PARAM_AA:
                    continue          # angle-axis never takes the general frame model
                for names, P in pose_sets(param, len(pts), path == "general", rng):
                    if offset:
                        P[:, :3, 3] -= P[:, :3, :3] @ np.full(3, offset)        # keep the clouds' world images near the origin
                    for cost in ([COST_P2P] if mode == "f32_no_normals" else costs):
                        for rk in robusts:
                            what = (tl, mode, path, param, cost, rk, offset, names)
                            wv, pinned = compare_blocks(eng, O, pts, nor, P, edges, corr, w, fixed, param, cost, ROBUST[rk], tl,
                                                        what, use_oracle)
                            worst = max(worst, wv)
                            if pinned:
                                oracle_sets.add((path, param))
    finally:
        eng.close()
    if use_oracle:                    # every parameterisation on every path has at least one set that pins the oracle
        want = {(p, q) for p in paths for q in params if not (p == "general" and q == PARAM_AA)}
        assert oracle_sets == want, (want - oracle_sets)
    return worst


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("tl", [1024, 8192])
def test_edge_blocks_match_extended_reference(oracle, tl, mode):
    # the tiny and huge weights change no slot arithmetic: at the 8192-slot tile the edges' own weights and no loss suffice
    run_block_cases(oracle, tl, mode, robusts=tuple(ROBUST) if tl == 1024 else ("off", "edge"), use_oracle=tl == 1024)


@pytest.mark.parametrize("offset", [1e3, 1e5])
def test_edge_blocks_far_from_origin(oracle, offset):
    """fp64 clouds 1e3 m and 1e5 m from their frames' origins: the bound scales with the magnitudes, the tolerance does not move."""
    run_block_cases(oracle, 1024, "f64", costs=[COST_P2P, COST_MIXED], robusts=("off", "edge"), offset=offset)


# ---- the readout itself ----------------------------------------------------------------------------------------------
def test_readout_state_and_last_evaluation(oracle):
    """No blocks before an LM evaluation or after the graph changed; the cost column sums to the summary's cost at the last
    evaluation: the start point after max_num_iterations = 0, the accepted point after one successful iteration (the
    evaluation enqueued behind the finished solve is skipped and leaves the blocks alone), and the rejected candidate after
    a step that fails (a frame turned 90 degrees from its matches and an initial radius of 1e16: the oracle's first step has
    rho < 0, and the blocks' cost is the oracle's candidate cost, not the kept start cost)."""
    pts, nor, edges, corr, w, _ = block_scene(1024)
    rng = np.random.default_rng(3)
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges)
    with pytest.raises(MvicpError):
        edge_blocks(eng)
    P0 = np.stack([np.eye(4)] * len(pts)); P0[:, :3, 3] = rng.uniform(-0.1, 0.1, (len(pts), 3))
    fx = _fixed_list(len(pts), (0,))
    eng.set_poses(P0, fx)
    for e in range(len(edges)):
        eng.set_edge(e, corr[e][0], corr[e][1], w[e])
    for iters in (0, 1):
        opt = default_options(); opt.max_num_iterations = iters
        s = eng.optimize(PARAM_SE3, COST_MIXED, True, options=opt)
        c = math.fsum(edge_blocks(eng)[:, 156])
        want = s["initial_cost"] if iters == 0 else s["final_cost"]
        assert s["num_successful_steps"] == iters and abs(c - want) <= 1e-12 * want, (iters, s, c)
        eng.set_poses(P0, fx)
    eng.set_graph(edges)
    with pytest.raises(MvicpError):
        edge_blocks(eng)
    eng.close()
    import test_gpu_lm_options as L
    pr = L.turned(L.ring_problem(oracle, 300), 2, 90)
    eopt, oopt = L.options(initial_trust_region_radius=1e16, max_num_iterations=1)
    _, sref, tr = pr.oracle(oracle, PARAM_AA, COST_MIXED, True, oopt)
    assert len(tr) == 2 and not tr[1, L.ACC] and tr[1, L.RHO] < -0.5, tr             # rejected, far from the 1e-3 threshold
    eng = Engine(); eng.set_frames(pr.pts, pr.nor); eng.set_graph(pr.edges); eng.set_poses(pr.poses, pr.fx)
    for e, (sf, _) in enumerate(pr.edges):
        if not pr.fx[sf]:
            eng.set_edge(e, pr.corr[e][0], pr.corr[e][1], pr.w[e])
    s = eng.optimize(PARAM_AA, COST_MIXED, True, options=eopt)
    c = math.fsum(edge_blocks(eng)[:, 156])
    assert s["num_successful_steps"] == 0 and s["num_iterations"] == 1 and s["final_cost"] == s["initial_cost"], s
    assert abs(c - tr[1, L.CAND]) <= 1e-9 * tr[1, L.CAND] and c > 1.2 * s["final_cost"], (s, c, tr[1])
    eng.close()


def test_readout_component_without_free_frame(oracle):
    """In a component solve, the edges of a component whose frames are all fixed belong to no problem and are never written:
    after a joint solve that filled them, the readout still returns zeros for them."""
    from helpers import oracle_correspond, scene
    from test_gpu_lm_graphs import _corr_of, topology
    M, edges, _ = topology("two_components")
    sc = scene(M, 1000, 43)
    corr, w = _corr_of(oracle_correspond(oracle, sc["pts"], sc["poses_init"], edges))
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges)
    for e in range(len(edges)):
        eng.set_edge(e, corr[e][0], corr[e][1], w[e])
    second = np.array([s >= 5 for s, _ in edges])
    eng.set_poses(sc["poses_init"], _fixed_list(M, (0, 5)))
    eng.optimize(PARAM_SE3, COST_P2PLANE, True)
    before = edge_blocks(eng)
    assert all(np.any(before[e]) for e in range(len(edges)) if edges[e][0] not in (0, 5))
    eng.set_poses(sc["poses_init"], _fixed_list(M, (0, 5, 6, 7, 8, 9)))
    summ = eng.optimize_components(PARAM_SE3, COST_P2PLANE, True)
    assert summ[1]["num_iterations"] == 0, summ
    after = edge_blocks(eng)
    assert not np.any(after[second]) and np.all(np.isfinite(after))
    assert all(np.any(after[e]) for e in range(len(edges)) if not second[e] and edges[e][0] != 0)
    eng.close()


# ---- outcome-level companion: solves through pi ------------------------------------------------------------------------
def pi_scene(n_views, start, truth, axes, n_points=1500, seed=11):
    """One cloud seen by n_views frames; frame f's true rotation truth(axis_f) and start rotation start(axis_f), frame 0 at the
    identity.  Identity matches on every edge of a ring with chords."""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-0.5, 0.5, (n_points, 3)); X[:, 2] *= 0.3
    N = rng.normal(size=(n_points, 3)); N /= np.linalg.norm(N, axis=1, keepdims=True)
    pts, nor, poses = [], [], []
    for f in range(n_views):
        Rt, Rs = (np.eye(3), np.eye(3)) if f == 0 else (truth(axes[f]), start(axes[f]))
        t = np.zeros(3) if f == 0 else rng.uniform(-0.1, 0.1, 3)
        pts.append(((X - t) @ Rt + rng.normal(0, 1e-3, X.shape)).astype(np.float32).astype(np.float64))
        nor.append((N @ Rt).astype(np.float32).astype(np.float64))
        P = np.eye(4); P[:3, :3] = Rs; P[:3, 3] = t
        poses.append(P)
    edges = [(i, j) for i in range(n_views) for j in range(n_views) if i != j]
    idx = np.arange(n_points, dtype=np.int32)
    corr = [(idx, idx) for _ in edges]
    w = [np.float32(0.05)] * len(edges)
    return pts, nor, np.stack(poses), edges, corr, w


PI_AXES = [None, (0.0, 0.6, 0.8), (1.0, 0.0, 0.0), (-0.48, 0.6, 0.64)]


@pytest.mark.parametrize("param", PARAMS)
@pytest.mark.parametrize("start", ["pi-5e-3", "pi"])
@pytest.mark.parametrize("path", ["unit", "general"])
def test_solve_through_pi_matches_oracle(oracle, param, start, path):
    """Frames that start at pi - 5e-3 (or exactly pi) about an axis and whose matches come from pi + 5e-3 about the same axis:
    the angle-axis iterates cross |w| = pi (the AA plus is plain addition).  Unit path in fp32 storage, general path
    (non-unit start poses) in fp64 storage."""
    if path == "general" and param == PARAM_AA:
        pytest.skip("angle-axis never takes the general frame model")
    th0 = math.pi - 5e-3 if start == "pi-5e-3" else math.pi
    axes = PI_AXES if start == "pi-5e-3" else [None, (1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0)]
    exact = {(1.0, 0.0, 0.0): np.diag([1.0, -1.0, -1.0]), (0.0, 1.0, 0.0): np.diag([-1.0, 1.0, -1.0]), (0.0, 0.0, 1.0): np.diag([-1.0, -1.0, 1.0])}
    startf = (lambda a: exact[a]) if start == "pi" else (lambda a: _rot(a, th0))
    pts, nor, poses, edges, corr, w = pi_scene(4, startf, lambda a: _rot(a, math.pi + 5e-3), axes)
    if path == "general":
        pts = [p + OFF_GRID for p in pts]
        poses[1:, :3, :3] *= 1 + 1e-3
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges)
    for cost in (COST_P2P, COST_P2PLANE):
        P, s, Pref, _ = compare_solve(oracle, eng, pts, nor, poses, edges, corr, w, param, cost, True, tag=("pi", start, path))
        assert TERMINATION[s["termination"]] != "NO_CONVERGENCE" and s["num_successful_steps"] > 0, s
    eng.close()
