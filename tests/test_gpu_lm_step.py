"""The LM step itself (csrc/lm_step.cuh, lm_step_body between the gathered blocks and the next candidate) against a damped solve
in numpy.longdouble, on one accepted first step per case.

Observation.  A solve with max_num_iterations = 0 from P0 leaves, in mvicp_debug_edge_blocks, the per-edge records the step
kernel gathers at x0 (a second such solve must return the same bits).  A solve with max_num_iterations = 1 and the same options
takes one step, which must be accepted; its poses are P1 = pose_of_param(x0 (+) delta).  From the engine's own records the
reference rebuilds, per problem, H and g over the free frames' local columns in ascending frame order (H from its lower
triangle, as the step reads it), and with them

    s_j = 1 / (1 + sqrt(H_jj))  (1 without Jacobi scaling),  D_j = clamp(s_j^2 H_jj, min_lm_diagonal, max_lm_diagonal),
    A = S H S + D / radius,  y = A^-1 S g,  delta = -S y,  x1 = x0 (+) delta,  P1_ref = pose_of_param(x1),

all in longdouble, x0 being the fp64 param_of_pose of test_gpu_lm_blocks.  Evaluation error is not part of this test (the
records are its input; test_gpu_lm_blocks pins them).

Bound, derived per entry (u = 2^-53, gamma_k = k u / (1 - k u)):
  gather     an entry of H or g summed from c list terms carries gamma_{c-1} times the sum of the terms' magnitudes (dH, dg);
  scale      s_j in relative error theta_j = gamma_3 + dH_jj / (2 (H_jj - dH_jj)) (1 + gamma_3): sqrt, add, divide, and the
             gathered H_jj (|ds / s| <= |dh| / 2h); 0 without scaling;
  products   s_i H_ij s_j in two roundings: |dA_ij| <= s_i s_j (dH_ij (1 + phi_ij) + |H_ij| phi_ij),
             phi_ij = (1 + theta_i)(1 + theta_j)(1 + gamma_2) - 1;
  damping    the unclamped s_j^2 H_jj moves by the same dA_jj; the clamp is monotone, so D moves by at most the larger of
             |clamp(w +- dA_jj) - D| (exactly 0 where the clamp binds on the whole interval); D / radius, sqrt and the square
             add gamma_4 of D / radius; the add onto the pivot u of the pivot;
  rhs        |d(s g)_j| <= s_j (dg_j (1 + theta_j)(1 + u) + |g_j| ((1 + theta_j)(1 + u) - 1));
  Cholesky   the factor, the forward substitution carried as row n and the back substitution are backward stable for any
             order of their sums: (A + dA + dC) y' = b + db, |dC| <= gamma_{3n+1} |L'| |L'^T| (Higham, Thm 10.4).  Where the
             theorem has one correctly rounded division or sqrt per entry, the engine multiplies by rsqrt's reciprocal pivot
             (1 ulp, <= 2u) and forms L_kk = d rsqrt(d): two more roundings in each of the factor, the forward and the back
             substitution, gamma_{3n+7}.  L' is the engine's factor; the longdouble factor L is used,
             times 1.01 (L' - L is of the order cond(A) u relative, below 1e-6 on every case here);
  fixed point  y' - y = A^-1 (db - (dA + dC) y'), so |y' - y| <= B for every B >= |A^-1| (|db| + (|dA| + |dC|)(|y| + B)); B is
             T^6(0) times 1.001 and T(B) <= B is asserted (a monotone map with T(B) <= B bounds every fixed point below it);
  step       delta' = y' s' in one rounding: |delta' - delta|_j <= s_j (B_j (1 + theta_j)(1 + u) + |y_j| ((1 + theta_j)(1 + u) - 1));
  x0         the engine's param_of_pose and its fp64 restatement each within gamma_12 of the formula: quaternion entries are
             at most 1 in magnitude (1.1 for the 1e-3 non-rigid scaling), angle-axis entries x kk with |x| <= 1; translations
             are copied exactly;
  (+), pose  F(x0, delta) = pose_of_param(x0 (+) delta) to first order through |dF / d delta| and |dF / d x0|, plus the
             rounding of (+) itself through |d pose / d x1| and pose_of_param's own rounding (gamma_4 of the quaternion
             matrix's magnitudes, 3 gamma_16 for Rodrigues with its 2-ulp sin / cos, translations exact).  The derivatives are
             the composed longdouble maps' central differences (h = 1e-6, times 1.001, plus 1e-11 (1 + |x|) + 4 u_ld (1 + |F|) / h
             absolute for the truncation and rounding of the difference); at delta = 0 they are the tangent derivatives D_j,
             c_j of test_gpu_lm_blocks.Frame, which is asserted on the unit path and the general quaternion path.  Second order: 32 (1 + |x|) (sum of the input perturbations)^2
             (every second derivative of these maps is below 64 (1 + |x|) on |delta| < 1).

Tightness.  Per group of cases the largest pose bound must stay below a stated threshold (well below the 1e-8 of the solve
tests), and the largest |delta_j| must be at least 1e-4: a bound that is always loose, or a step that is nearly zero, proves
nothing.  The threshold is not applied to the ill-conditioned case (cond(A) >= 1e8), whose bound must still close and hold.

Which branches the cases reach: the envelope shapes of test_gpu_lm_graphs (loop closure, a hub on the last frame, random
graphs, frames that are only a dst, a fixed dst in the middle, two components in one solve), a chain (tridiagonal), a star into
fixed frame 0 (block diagonal: the trailing update touches only the rhs row, the look-ahead has nothing to update), one free
frame (n = 6, no look-ahead), and the wide graphs whose factor stays in shared memory (36 views) or goes to global memory
(48 views); every parameterisation on the unit path and the quaternion ones on the general path; the trust-region options,
including the clamps, which are the only cases where the Jacobi scale reaches the step (without a binding clamp
delta = -(H + diag(H) / radius)^-1 g whatever the scale); a rejected step followed by an accepted one at half the radius with
the reused diagonal; a component batch with the factor in shared memory for some CTAs and in global memory for another."""
import math

import numpy as np
import pytest

import test_gpu_lm_blocks as B
import test_gpu_lm_graphs as G
from helpers import oracle_correspond, scene
from mv_lm_icp_b200 import COST_MIXED, COST_P2P, COST_P2PLANE, PARAM_AA, PARAM_QUAT, PARAM_SE3, Engine, synth
from mv_lm_icp_b200.api import TERMINATION, default_options
from test_gpu_g2o_blocks import _chol_ld, _chol_solve_ld

pytestmark = pytest.mark.gpu
LD = np.longdouble
U = B.U
U_LD = LD(np.finfo(LD).eps) / 2
gamma = B.gamma
# Largest pose bound per group (set from the bound's value on the cases, never from the errors).  Graphs of up to 14 views:
# their steps reach 0.24 rad, and the Cholesky's gamma_{3n+7} |A^-1| |L| |L^T| |y| puts the bound at 3e-12 ... 5e-11 (about
# 1e-11 on the 5-view ring of the trust-region cases).  The wide graphs and the component batch with 48 views: at n = 210
# and 282 the same term gives 4e-10 ... 6e-10 (a frame of the wide graph turns by 0.2 rad); the bound would need the
# envelope's inner-product lengths in place of n to come down, which the graphs' full-width rows do not offer.  Clouds 1e5 m
# from the origin, where the rounding of t + dt alone is ~1e-11.
LIMIT = {"small": 6e-11, "wide": 1e-9, "far": 1e-10}


# ---- longdouble (+) and pose_of_param ----------------------------------------------------------------------------------
def _quat_matrix(q):
    """matrix_of_quat: the polynomial map I + 2 w [u]x + 2 [u]x^2 (a rotation only for a unit q)."""
    Uq = B._skew(q[:3])
    return np.eye(3, dtype=LD) + 2 * q[3] * Uq + 2 * Uq @ Uq


def plus_ld(param, x, d):
    """param_plus: angle-axis x + d; quaternion [sin|d| d / |d|, cos|d|] (x) q and t + dt; SE3 x * exp(d), renormalised."""
    x = np.asarray(x, LD); d = np.asarray(d, LD)
    if param == PARAM_AA:
        return x + d
    if param == PARAM_QUAT:
        n2 = d[:3] @ d[:3]
        sinc = B._trig(n2)[0]
        dq = np.concatenate([sinc * d[:3], [np.cos(np.sqrt(n2))]])
        return np.concatenate([B._quat_prod(dq, x[:4]), x[4:] + d[3:]])
    w = d[3:]; th2 = w @ w
    sinc_h = B._trig(th2 / 4)[0]                       # sin(th / 2) / (th / 2)
    qe = np.concatenate([sinc_h / 2 * w, [np.cos(np.sqrt(th2) / 2)]])
    _, c1, c2 = B._trig(th2)
    W = B._skew(w)
    te = (np.eye(3, dtype=LD) + c1 * W + c2 * W @ W) @ d[:3]
    q = B._quat_prod(x[:4], qe)
    q = q / np.sqrt(q @ q)
    return np.concatenate([q, x[4:] + _quat_matrix(x[:4]) @ te])


def pose_ld(param, x):
    """pose_of_param as a 3x4 [R | t]: Rodrigues (I + [w]x at th^2 <= DBL_EPSILON), or the quaternion's polynomial map."""
    x = np.asarray(x, LD)
    if param == PARAM_AA:
        w = x[:3]; th2 = w @ w; W = B._skew(w)
        if th2 > B.EPS:
            sinc, a, _ = B._trig(th2)
            R = np.eye(3, dtype=LD) + sinc * W + a * W @ W
        else:
            R = np.eye(3, dtype=LD) + W
        return np.concatenate([R, x[3:, None]], 1)
    return np.concatenate([_quat_matrix(x[:4]), x[4:, None]], 1)


H_FD = LD(1e-6)


def _jac(f, v):
    """|central differences| of f (-> 12) over the entries of v, times 1.001, plus the difference's truncation and rounding."""
    v = np.asarray(v, LD)
    cols, top = [], LD(0)
    for i in range(len(v)):
        e = np.zeros(len(v), LD); e[i] = H_FD
        a, b = f(v + e), f(v - e)
        top = max(top, np.max(np.abs(a)), np.max(np.abs(b)))
        cols.append((a - b) / (2 * H_FD))
    J = np.stack(cols, 1)
    return J, np.abs(J) * LD(1.001) + LD(1e-11) * (1 + np.max(np.abs(v))) + 4 * U_LD * (1 + top) / H_FD


def _quat_prod_abs(a, b):
    """The quaternion product of |a| and |b| with every term added: the magnitude of quat_prod's sums."""
    s = np.sum(a[:3] * b[:3])
    return np.array([a[3] * b[0] + a[0] * b[3] + a[1] * b[2] + a[2] * b[1], a[3] * b[1] + a[1] * b[3] + a[2] * b[0] + a[0] * b[2],
                     a[3] * b[2] + a[2] * b[3] + a[0] * b[1] + a[1] * b[0], a[3] * b[3] + s])


def _rounding_plus(param, x0, d, x1):
    """|fl(x0 (+) d) - (x0 (+) d)| per ambient entry, from the magnitudes of param_plus's operations."""
    if param == PARAM_AA:
        return gamma(1) * (np.abs(x0) + np.abs(d))
    out = np.zeros(7, LD)
    if param == PARAM_QUAT:       # dq: sqrt, sin (2 ulp), divide, multiply; the product 4 terms: gamma_12 of |dq| (x) |q|
        n = np.sqrt(d[:3] @ d[:3])
        dq = np.concatenate([np.abs(d[:3]) * (abs(np.sin(n) / n) if n > 0 else 1), [abs(np.cos(n))]])
        out[:4] = gamma(12) * _quat_prod_abs(dq, np.abs(x0[:4]))
        out[4:] = gamma(1) * (np.abs(x0[4:]) + np.abs(d[3:]))
        return out
    # SE3: exp (sin / cos 2 ulp, the cancellations 1 - cos and th - sin counted at |cos| + 1 and th + |sin|), V upsilon,
    # the product and its normalisation, then t0 + F(q0) te
    w = d[3:]; th = np.sqrt(w @ w); Wm = np.abs(B._skew(w))
    if th >= 1e-10:
        c1m, c2m = (1 + abs(np.cos(th))) / th ** 2, (th + abs(np.sin(th))) / th ** 3
        te_m = (np.eye(3, dtype=LD) + c1m * Wm + c2m * Wm @ Wm) @ np.abs(d[:3])
    else:
        te_m = 3 * np.abs(d[:3]) + np.sum(np.abs(d[:3]))
    q0m = np.abs(x0[:4]); Um = np.abs(B._skew(q0m[:3]))
    Fm = np.eye(3, dtype=LD) + 2 * q0m[3] * Um + 2 * Um @ Um
    out[:4] = gamma(24) * (1 + np.sum(q0m))
    out[4:] = gamma(1) * (np.abs(x0[4:]) + Fm @ te_m) + gamma(24) * (Fm @ te_m)
    return out


def _rounding_pose(param, x1):
    R = np.zeros((3, 4), LD)
    if param == PARAM_AA:
        R[:, :3] = 3 * gamma(16)
    else:
        qm = np.abs(x1[:4]); Um = np.abs(B._skew(qm[:3]))
        R[:, :3] = gamma(4) * (np.eye(3, dtype=LD) + 2 * qm[3] * Um + 2 * Um @ Um)
    return R


def _x0_error(param, x0):
    """|engine param_of_pose - fp64 restatement| per ambient entry (translations are copied)."""
    out = np.zeros(len(x0), LD)
    if param == PARAM_AA:
        th = float(np.linalg.norm(x0[:3]))
        kk = 2 * th / math.sin(th / 2) if th > 0 else 2.0
        out[:3] = 2 * gamma(12) * max(kk, 2.0)
    else:
        out[:4] = 2 * gamma(12) * max(1.1, float(np.max(np.abs(x0[:4]))))
    return out


def frame_check(param, x0, d, Bd, dx0):
    """(P1_ref 3x4, bound 3x4) for one free frame from x0 (fp64), delta (ld) and their bounds."""
    x0l = np.asarray(x0, LD)
    x1 = plus_ld(param, x0l, d)
    P = pose_ld(param, x1)
    F = lambda a, b: pose_ld(param, plus_ld(param, a, b)).ravel()          # noqa: E731
    _, Jd = _jac(lambda v: F(x0l, v), d)
    _, Jx = _jac(lambda v: F(v, d), x0l)
    _, Jp = _jac(lambda v: pose_ld(param, v).ravel(), x1)
    dx1 = _rounding_plus(param, x0l, d, x1)
    tot = np.sum(Bd) + np.sum(dx0) + np.sum(dx1)
    second = 32 * (1 + np.max(np.abs(x1))) * tot * tot
    bound = (Jd @ Bd + Jx @ dx0 + Jp @ dx1 + second).reshape(3, 4) + _rounding_pose(param, x1)
    return P, bound


def check_tangent_derivatives(param, x):
    """At delta = 0 the central differences of pose(x (+) delta) are test_gpu_lm_blocks.Frame's D_j and c_j."""
    fr = B.Frame(param, x)
    J, _ = _jac(lambda v: pose_ld(param, plus_ld(param, np.asarray(x, LD), v)).ravel(), np.zeros(6, LD))
    for j in range(6):       # (on the unit path: a non-unit SE3 x (+) 0 is renormalised, Frame differentiates at x as Ceres does)
        want = np.concatenate([fr.D[j], fr.c[j][:, None]], 1).ravel()
        assert np.max(np.abs(J[:, j] - want)) <= 1e-9 * (1 + np.max(np.abs(x))), (param, j)


# ---- the normal equations of one problem from the engine's records -------------------------------------------------------
def assemble(rec, edges, frames, fx, pedges):
    """H (lower triangle mirrored), g, and per entry the sum of its terms' magnitudes and the term count, over the free frames
    of `frames` (ascending) in their local columns; pedges: the problem's edges in graph order."""
    col, n = {}, 0
    for f in frames:
        if not fx[f]:
            col[f] = n; n += 6
    H, Hm = np.zeros((n, n), LD), np.zeros((n, n), LD)
    g, gm = np.zeros(n, LD), np.zeros(n, LD)
    Hc, gc = np.zeros((n, n), int), np.zeros(n, int)
    for e in pedges:
        s, k = edges[e]
        if fx[s]:
            assert not np.any(rec[e]), ("an edge of a fixed src holds a record", e)
            continue
        Hp = rec[e, :144].reshape(12, 12).astype(LD); gp = rec[e, 144:156].astype(LD)
        sides = [(col[s], 0)] + ([(col[k], 6)] if not fx[k] else [])
        for ca, oa in sides:
            g[ca:ca + 6] += gp[oa:oa + 6]; gm[ca:ca + 6] += np.abs(gp[oa:oa + 6]); gc[ca:ca + 6] += 1
            for cb, ob in sides:
                blk = Hp[oa:oa + 6, ob:ob + 6]
                H[ca:ca + 6, cb:cb + 6] += blk; Hm[ca:ca + 6, cb:cb + 6] += np.abs(blk); Hc[ca:ca + 6, cb:cb + 6] += 1
    low = np.tril(np.ones((n, n), bool))
    H = np.where(low, H, H.T); Hm = np.where(low, Hm, Hm.T); Hc = np.where(low, Hc, Hc.T)
    return col, H, g, Hm, Hc, gm, gc


def _gam(c):
    c = np.asarray(c, LD)
    return c * U / (1 - c * U)


def solve_reference(H, g, Hm, Hc, gm, gc, opt, radius):
    """The damped solve in longdouble and the componentwise bound of the module docstring.  Returns a dict."""
    n = len(g)
    r = LD(radius)
    dH = _gam(np.maximum(Hc - 1, 0)) * Hm + Hc * U_LD * Hm         # the gather, and the reference's own longdouble sums
    dg = _gam(np.maximum(gc - 1, 0)) * gm + gc * U_LD * gm
    h, dh = np.diag(H).copy(), np.diag(dH).copy()
    if opt.jacobi_scaling:
        assert np.all(h > 2 * dh), "a pivot without residuals"
        s = 1 / (1 + np.sqrt(h))
        th = gamma(3) + dh / (2 * (h - dh)) * (1 + gamma(3))
    else:
        s, th = np.ones(n, LD), np.zeros(n, LD)
    phi = np.outer(1 + th, 1 + th) * (1 + gamma(2)) - 1
    A = np.outer(s, s) * H
    dA = np.outer(s, s) * (dH * (1 + phi) + np.abs(H) * phi)
    w, dw = s * s * h, np.diag(dA).copy()
    mn, mx = LD(opt.min_lm_diagonal), LD(opt.max_lm_diagonal)
    D = np.clip(w, mn, mx)
    dD = np.maximum(np.abs(np.clip(w + dw, mn, mx) - D), np.abs(np.clip(w - dw, mn, mx) - D))
    A[np.diag_indices(n)] += D / r
    dA[np.diag_indices(n)] += dD / r * (1 + gamma(4)) + D / r * gamma(4)
    dA[np.diag_indices(n)] += U * (np.diag(A) + np.diag(dA))
    b = s * g
    db = s * (dg * (1 + th) * (1 + U) + np.abs(g) * ((1 + th) * (1 + U) - 1))
    L = _chol_ld(A)
    y = _chol_solve_ld(L, b)
    Ainv = np.stack([_chol_solve_ld(L, e) for e in np.eye(n, dtype=LD)], 1)
    aL = np.abs(L)
    dT = dA + gamma(3 * n + 7) * LD(1.01) * (aL @ aL.T)
    aAinv = np.abs(Ainv)
    T = lambda Bv: aAinv @ (db + dT @ (np.abs(y) + Bv))        # noqa: E731
    Bv = np.zeros(n, LD)
    for _ in range(6):
        Bv = T(Bv)
    Bv = Bv * LD(1.001)
    assert np.all(T(Bv) <= Bv), "the step's perturbation bound does not close"
    delta = -s * y
    Bd = s * (Bv * (1 + th) * (1 + U) + np.abs(y) * ((1 + th) * (1 + U) - 1))
    cond = float(np.max(np.sum(np.abs(A), 1)) * np.max(np.sum(aAinv, 1)))
    return dict(delta=delta, Bd=Bd, w=w, dw=dw, D=D, A=A, cond=cond, s=s, n=n)


# ---- one case ------------------------------------------------------------------------------------------------------------
def _options(over, max_iter):
    o = default_options()
    for k, v in over.items():
        setattr(o, k, v)
    o.max_num_iterations = max_iter
    return o


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def run_step(eng, P0, fx, edges, problems, param, cost, robust, over=None, what="", components=False, limit=None,
             after=None, reject_first=False):
    """Solve with max_num_iterations = 0 twice (the records, the parameter round trip of P0), then 1 (2 with reject_first:
    one rejected step, then the step at half the radius with the reused diagonal), and hold every free frame of every
    problem to its reference.  problems: [(frames ascending, edges in graph order)].  over: option overrides (a callable
    value is resolved from the first problem's reference at the default options).  after(refs): extra assertions.
    Returns the per-problem references."""
    over = dict(over or {})
    solve = (lambda o: eng.optimize_components(param, cost, robust, options=o)) if components else \
        (lambda o: [eng.optimize(param, cost, robust, options=o)])
    recs = []
    for _ in range(2):
        eng.set_poses(P0, fx)
        s0 = solve(_options({k: v for k, v in over.items() if not callable(v)}, 0))
        assert all(TERMINATION[s["termination"]] == "MAX_ITERATIONS" for s in s0 if s["num_evaluations"]), (what, s0)
        recs.append(B.edge_blocks(eng))
    assert np.array_equal(_bits(recs[0]), _bits(recs[1])), (what, "the records are not reproducible")
    rec = recs[0]
    P_rt = eng.get_poses()
    asm = [assemble(rec, edges, fr, fx, pe) for fr, pe in problems]
    for k, v in list(over.items()):
        if callable(v):
            c0 = asm[0]
            ref0 = solve_reference(*c0[1:], _options({}, 1), default_options().initial_trust_region_radius)
            over[k] = float(v(ref0))
    opt = _options(over, 2 if reject_first else 1)
    if reject_first:
        eng.set_poses(P0, fx)
        s1 = solve(_options(over, 1))
        assert all(s["num_successful_steps"] == 0 and s["num_iterations"] == 1 for s in s1), (what, s1)
        assert np.array_equal(_bits(eng.get_poses()), _bits(P_rt)), (what, "a rejected step moved a pose")
    eng.set_poses(P0, fx)
    summ = solve(opt)
    P1 = eng.get_poses()
    want_it = 2 if reject_first else 1
    refs, top, worst, emax, dmax, bmax = [], 0.0, 0.0, 0.0, 0.0, 0.0
    for (frames, _), (col, H, g, Hm, Hc, gm, gc), s in zip(problems, asm, summ):
        if not col:
            continue
        assert s["num_iterations"] == want_it and s["num_successful_steps"] == 1, (what, s)
        radius = opt.initial_trust_region_radius / (2 if reject_first else 1)
        ref = solve_reference(H, g, Hm, Hc, gm, gc, opt, radius)
        refs.append(ref)
        for f in frames:
            if f not in col:
                assert np.array_equal(_bits(P1[f]), _bits(P_rt[f])), (what, f, "a fixed frame moved")
                continue
            c0 = col[f]
            x0 = B.param_of_pose(param, P0[f])
            Pref, bound = frame_check(param, x0, ref["delta"][c0:c0 + 6], ref["Bd"][c0:c0 + 6], _x0_error(param, x0))
            err = np.abs(P1[f][:3].astype(LD) - Pref)
            assert np.array_equal(P1[f][3], [0, 0, 0, 1]), (what, f)
            ratio = err / bound
            i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
            assert np.all(err <= bound), (what, f, "out of bound", i, float(P1[f][:3][i]), float(Pref[i]), float(err[i]),
                                          float(bound[i]))
            worst = max(worst, float(np.max(ratio))); top = max(top, float(np.max(bound))); emax = max(emax, float(np.max(err)))
        dmax = max(dmax, float(np.max(np.abs(ref["delta"])))); bmax = max(bmax, float(np.max(ref["Bd"])))
    assert refs, what
    cond = max(r["cond"] for r in refs)
    print(f"{what}: n {[r['n'] for r in refs]}, cond(A) {cond:.3g}, |delta| up to {dmax:.3g}, step bound {bmax:.3g}, "
          f"largest pose bound {top:.3g}, largest error {emax:.3g}, worst error / bound {worst:.3g}")
    assert dmax >= 1e-4, (what, "the step is trivially small", dmax)
    if limit is not None:
        assert top <= LIMIT[limit], (what, "the bound is loose", top, LIMIT[limit])
    if after:
        after(refs)
    return refs


# ---- scenes ------------------------------------------------------------------------------------------------------------
def load(O, pts, nor, poses, edges, fixed, corr=None, w=None):
    """Engine with frames, graph and the oracle's correspondences at `poses` (edges of a fixed src are not uploaded)."""
    fx = G._fixed_list(len(pts), fixed)
    if corr is None:
        corr, w = G._corr_of(oracle_correspond(O, pts, poses, edges))
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges)
    eng.set_poses(poses, fx)
    for e, (s, _) in enumerate(edges):
        if not fx[s]:
            eng.set_edge(e, corr[e][0], corr[e][1], w[e])
    return eng, fx


def graph_scene(M, n_points=1000, cfg=43, views=None, path="unit"):
    sc = scene(M, n_points, cfg)
    order = list(range(M)) if views is None else [views.index(f) for f in range(M)]
    pts, nor = [sc["pts"][v] for v in order], [sc["nor"][v] for v in order]
    poses = sc["poses_init"][order].copy()
    if path == "general":
        poses[1] = G._nonrigid(poses[1])
        poses[3] = G._nonrigid(poses[3])
    return pts, nor, poses


def joint(O, M, edges, fixed=(0,), param=PARAM_SE3, cost=COST_P2PLANE, robust=True, over=None, what="", limit="small",
          n_points=1000, cfg=43, views=None, path="unit", after=None):
    pts, nor, poses = graph_scene(M, n_points, cfg, views, path)
    eng, fx = load(O, pts, nor, poses, edges, fixed)
    try:
        return run_step(eng, poses, fx, edges, [(list(range(M)), list(range(len(edges))))], param, cost, robust, over, what,
                        limit=limit, after=after)
    finally:
        eng.close()


def chain_edges(M):
    return [(i + 1, i) for i in range(M - 1)] + [(i, i + 1) for i in range(M - 1)]


def star_edges(M):
    return [(i, 0) for i in range(1, M)]


def _starts_at_own_block(M, edges, fixed):
    rfirst, n = G.row_profile(M, edges, fixed)
    return all(rfirst[r] == (r // 6) * 6 for r in range(n))


SHAPES = ["ring_chord", "hub_last", "random1", "random2", "random3", "dst_only", "dst_fixed", "two_components", "chain", "star",
          "single", "wide36", "wide48"]


def shape(name):
    """(M, edges, fixed, views, limit group) of an envelope shape."""
    if name == "chain":
        M, edges = 6, chain_edges(6)
        rfirst, n = G.row_profile(M, edges, (0,))
        assert all(rfirst[r] == max(0, (r // 6 - 1) * 6) for r in range(n))         # tridiagonal blocks
        return M, edges, (0,), None, "small"
    if name == "star":                # block diagonal: every row starts at its own block, rlast = j0 + 5
        M, edges = 6, star_edges(6)
        assert _starts_at_own_block(M, edges, (0,))
        return M, edges, (0,), None, "small"
    if name == "single":
        return 2, [(1, 0), (0, 1)], (0,), None, "small"
    if name.startswith("wide"):
        M = int(name[4:])
        edges = G.wide_graph(M)
        need, _ = G.skyline_bytes(M, edges, (0,))
        assert (need > G.SMEM_LIMIT) == (M == 48), need
        return M, edges, (0,), None, "wide"
    M, edges, fixed = G.topology(name)
    return M, edges, fixed, G.HUB_RING if name == "hub_last" else None, "small"


def check_shape(O, name, n_points=1000):
    M, edges, fixed, views, grp = shape(name)
    joint(O, M, edges, fixed, what=("shape", name), limit=grp, n_points=600 if M > 14 else n_points, views=views)


PARAM_CASES = [("aa", PARAM_AA, COST_P2PLANE, True, "unit"), ("quat", PARAM_QUAT, COST_P2PLANE, True, "unit"),
               ("se3", PARAM_SE3, COST_P2PLANE, True, "unit"), ("quat-general", PARAM_QUAT, COST_P2PLANE, True, "general"),
               ("se3-general", PARAM_SE3, COST_P2PLANE, True, "general"), ("quat-mixed", PARAM_QUAT, COST_MIXED, False, "unit"),
               ("aa-p2p", PARAM_AA, COST_P2P, True, "unit")]


def check_param(O, name, n_points=1000):
    _, param, cost, robust, path = next(c for c in PARAM_CASES if c[0] == name)
    M, edges, fixed = G.topology("ring_chord")
    pts, nor, poses = graph_scene(M, n_points, 43, None, path)
    if path == "unit" or param == PARAM_QUAT:
        check_tangent_derivatives(param, B.param_of_pose(param, poses[1]))
    joint(O, M, edges, fixed, param, cost, robust, what=("param", name), n_points=n_points, path=path)


# ---- trust-region settings --------------------------------------------------------------------------------------------
def _median_w(ref):
    return float(np.median(ref["w"]))


def _binds(low):
    """The clamp binds on some columns and not on others (with the bound on the unclamped value taken into account)."""
    def after(refs):
        r = refs[0]
        w, dw, D = r["w"], r["dw"], r["D"]
        hit = (w + dw < D) if low else (w - dw > D)
        free = np.abs(w - D) <= dw
        assert hit.any() and free.any() and (~hit).any(), ("clamp", low, int(hit.sum()), int(free.sum()))
    return after


TINY = 5e-3


def _diagonal_dominates(refs):
    """Every pivot's damping D_j / radius exceeds the rest of its row of A several times over."""
    A, D = refs[0]["A"], refs[0]["D"]
    rest = np.sum(np.abs(A), 1) - D / LD(TINY)
    ratio = float(np.min(D / LD(TINY) / rest))
    assert ratio > 3, ("the damping does not dominate", ratio)


TRUST = {
    "defaults": ({}, None),
    "gauss_newton": ({"initial_trust_region_radius": 1e16, "max_trust_region_radius": 1e16}, None),
    "tiny_radius": ({"initial_trust_region_radius": TINY}, _diagonal_dominates),
    "no_scaling": ({"jacobi_scaling": 0}, None),
    "min_diag_binds": ({"min_lm_diagonal": _median_w}, _binds(True)),
    "max_diag_binds": ({"max_lm_diagonal": _median_w}, _binds(False)),
    "min_diag_zero": ({"min_lm_diagonal": 0.0}, None),
}


def check_trust(O, name, n_points=1000):
    over, after = TRUST[name]
    M = 5
    for param in (PARAM_SE3, PARAM_QUAT):
        joint(O, M, synth.ring_edges(M, 2), (0,), param, COST_P2PLANE, True, over=over, what=("trust", name, param),
              n_points=n_points, cfg=61, after=after)


# ---- rejected, then accepted ----------------------------------------------------------------------------------------------
def check_reject_then_accept(O, n_points=1000):
    """test_gpu_lm_options' rejection scene (frame 2 turned 90 degrees from its matches): the first radius of the list
    whose first step is rejected and whose second (at half the radius, reused diagonal) is accepted."""
    import test_gpu_lm_options as Lo
    pr = Lo.turned(Lo.ring_problem(O, n_points), 2, 90)
    eng, fx = load(O, pr.pts, pr.nor, pr.poses, pr.edges, (0,), pr.corr, pr.w)
    try:
        for r0 in (1e16, 1e4, 1e3, 1e2, 30.0, 10.0, 3.0, 1.0, 0.3, 0.1):
            outs = []
            for k in (1, 2):
                eng.set_poses(pr.poses, fx)
                outs.append(eng.optimize(PARAM_QUAT, COST_P2PLANE, True, options=_options({"initial_trust_region_radius": r0}, k)))
            if outs[0]["num_successful_steps"] == 0 and outs[1]["num_successful_steps"] == 1:
                break
        else:
            pytest.fail("no radius in the list gives a rejection followed by an acceptance")
        run_step(eng, pr.poses, fx, pr.edges, [(list(range(len(pr.pts))), list(range(len(pr.edges))))], PARAM_QUAT,
                 COST_P2PLANE, True, {"initial_trust_region_radius": r0}, ("reject then accept", r0), limit="small",
                 reject_first=True)
    finally:
        eng.close()


# ---- a component batch ------------------------------------------------------------------------------------------------------
def check_components(O, n_points=800, wide=True):
    """A star into its lowest frame (fixed by the call: block-diagonal H), a ring, a two-frame pair and (wide) the 48-view
    component whose factor is in global memory, in one optimize_components call; each held to its own solve."""
    import test_gpu_components as T
    comps = [T.Comp(O, 5, star_edges(5), n_points=n_points, cfg=21), T.Comp(O, 6, synth.ring_edges(6, 2), n_points=n_points, cfg=22),
             T.Comp(O, 2, [(1, 0), (0, 1)], n_points=n_points, cfg=23)]
    assert _starts_at_own_block(5, star_edges(5), (0,))
    if wide:
        assert G.skyline_bytes(48, G.wide_graph(48), (0,))[0] > G.SMEM_LIMIT
        assert all(G.skyline_bytes(c.n, c.edges, (0,))[0] < G.SMEM_LIMIT for c in comps)
        comps.append(T.Comp(O, 48, G.wide_graph(48), n_points=600, cfg=24))
    b = T.Batch(comps)
    eng = Engine()

    def corr(e):
        k, r = b.emap[e]
        return b.comps[k].corr[r][0], b.comps[k].corr[r][1], b.comps[k].w[r]
    T._load(eng, b.pts, b.nor, b.poses, b.fx, b.edges, corr, "f32")
    problems = [(list(b.gid[k]), [e for e in range(len(b.edges)) if b.emap[e][0] == k]) for k in range(len(comps))]
    try:
        run_step(eng, b.poses, b.fx, b.edges, problems, PARAM_SE3, COST_P2PLANE, True, None, ("components", len(comps)),
                 components=True, limit="wide" if wide else "small")
    finally:
        eng.close()


# ---- ill-conditioned, far from the origin -------------------------------------------------------------------------------
def planar_scene(n_points=1200, curvature=1e-2, seed=5):
    """Two frames that see the same gently curved patch z = curvature (x^2 + 3 y^2) with its exact normals: under
    point-to-plane the in-plane motions are observable only through the curvature (the rotation about the normal through
    its anisotropy), cond(A) ~ 1 / curvature^2."""
    rng = np.random.default_rng(seed)
    xy = rng.uniform(-0.5, 0.5, (n_points, 2))
    X = np.concatenate([xy, curvature * (xy[:, :1] ** 2 + 3 * xy[:, 1:] ** 2)], 1)
    N = np.concatenate([-2 * curvature * xy[:, :1], -6 * curvature * xy[:, 1:], np.ones((n_points, 1))], 1)
    N /= np.linalg.norm(N, axis=1, keepdims=True)
    P1 = np.eye(4); P1[:3, :3] = G._rigid(np.random.default_rng(seed + 1), 1e-4, 0)[:3, :3]; P1[:3, 3] = [3e-3, -4e-3, 2e-3]
    X1 = (X - P1[:3, 3]) @ P1[:3, :3]
    pts = [X.astype(np.float32).astype(np.float64), X1.astype(np.float32).astype(np.float64)]
    nor = [N.astype(np.float32).astype(np.float64), (N @ P1[:3, :3]).astype(np.float32).astype(np.float64)]
    idx = np.arange(n_points, dtype=np.int32)
    return pts, nor, np.stack([np.eye(4), np.eye(4)]), [(1, 0)], [(idx, idx)], [np.float32(0.05)]


def check_ill_conditioned(O, n_points=1200):
    pts, nor, poses, edges, corr, w = planar_scene(n_points)
    eng, fx = load(O, pts, nor, poses, edges, (0,), corr, w)

    def cond_at_least(refs):
        assert refs[0]["cond"] >= 1e8, refs[0]["cond"]
    try:
        run_step(eng, poses, fx, edges, [([0, 1], [0])], PARAM_SE3, COST_P2PLANE, False,
                 {"min_lm_diagonal": 0.0, "initial_trust_region_radius": 1e16, "max_trust_region_radius": 1e16},
                 ("ill-conditioned",), limit=None, after=cond_at_least)
    finally:
        eng.close()


def check_far(O, param, offset=1e5, n_points=1000):
    """fp64 clouds `offset` from their frames' origins, world images where they were: the rounding of (+) and pose_of_param
    at |t| ~ offset dominates the bound."""
    M = 4
    edges = synth.ring_edges(M, 2)
    pts, nor, poses = graph_scene(M, n_points, 61)
    corr, w = G._corr_of(oracle_correspond(O, pts, poses, edges))
    pts = [p + offset + G.OFF_GRID for p in pts]
    poses = poses.copy()
    poses[:, :3, 3] -= poses[:, :3, :3] @ np.full(3, offset)
    assert not G._f32_exact(np.concatenate(pts))
    eng, fx = load(O, pts, nor, poses, edges, (0,), corr, w)
    try:
        run_step(eng, poses, fx, edges, [(list(range(M)), list(range(len(edges))))], param, COST_P2PLANE, True, None,
                 ("far", offset, param), limit="far")
    finally:
        eng.close()


# ---- the tests ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [c[0] for c in PARAM_CASES])
def test_step_parameterisations_and_paths(oracle, name):
    check_param(oracle, name)


@pytest.mark.parametrize("name", SHAPES)
def test_step_envelope_shapes(oracle, name):
    check_shape(oracle, name)


@pytest.mark.parametrize("name", list(TRUST))
def test_step_trust_region_settings(oracle, name):
    check_trust(oracle, name)


def test_step_rejected_then_accepted(oracle):
    check_reject_then_accept(oracle)


def test_step_component_batch(oracle):
    check_components(oracle)


def test_step_ill_conditioned(oracle):
    check_ill_conditioned(oracle)


@pytest.mark.parametrize("param", [PARAM_AA, PARAM_QUAT])
def test_step_far_from_origin(oracle, param):
    check_far(oracle, param)
