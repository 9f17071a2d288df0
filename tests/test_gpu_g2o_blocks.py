"""Per-edge normal equations of the g2o solve (g2o_eval_kernel + g2o_edge_kernel) against an extended-precision evaluation of
Edge_V_V_GICP, read edge by edge with mvicp_debug_edge_blocks after mvicp_optimize_g2o / mvicp_optimize_g2o_components.

Reference.  Per correspondence (first, second) of edge src -> dst, in numpy.longdouble (64-bit mantissa on x86-64), written
out here rather than taken from tests/g2o_model.py: vertex 0 = dst (F0, t0), vertex 1 = src (F1, t1), p = src point, q = dst
point, n = dst normal;
    e     = F0^T (F1 p + t1) - F0^T t0 - q          (Eigen's isometry inverse, also for a non-rigid F0)
    Omega = I, or R0^T diag(eps, eps, 1) R0 with R0 from makeRot0: row 2 = n (not normalised), row 1 = normalise((0,1,0) -
            n_y n) (a zero vector stays zero), row 0 = n x row 1
    J_dst = [-I | 2 [u]x],  J_src = [M01 | -2 M01 [p]x],  u = e + q,  M01 = F0^T F1
and per edge the pair matrix J^T Omega J over [src | dst], the gradient J^T Omega e and chi2 = sum e^T Omega e.

Tolerance.  Not fitted: every entry satisfies |engine - reference| <= gamma_k * magnitude, gamma_k = k u / (1 - k u), u = 2^-53.
The magnitude is the engine's own formulation redone in magnitude arithmetic (absolute values, subtractions as additions):
thread 0's F0^T, -F0^T t0 and M01; y = F1 p + t1, u, r; g2o_prec0 with its normalisation, which carries the relative
condition |y|_m / |y| of the vector it normalises (near n = +-e_y, 1 - n_y^2 cancels; there the subtraction is exact and
y_1's magnitude is the rounding of n_y^2, see prec0, so those normals keep a rounding-level bound); W = Omega J and the sums J^T W, J^T Omega r, r^T Omega r.  k (`k_depth`) is counted: the operation
depth per correspondence (K_CORR), the tile_len / 128 slots each lane pair accumulates, the xor tree (4), the 8 warps, and the
edge's tiles summed in order by g2o_edge_kernel.  Device FMA contraction only removes roundings, so the bound covers it."""
import ctypes as C
import math

import numpy as np
import pytest

import g2o_model as G
from mv_lm_icp_b200 import COST_P2P, COST_P2PLANE, PARAM_SE3, Engine, MvicpError, default_g2o_options, synth
from test_gpu_g2o import BUMP, synthetic
from test_gpu_g2o_graphs import fixed_flags, g2o_tile_scene, readout_options, upload
from test_gpu_lm_graphs import MODES, OFF_GRID, _f32_exact, _fixed_list, tile_len

LD = np.longdouble
EOUT = 160
U = 2.0 ** -53
EVAL_THREADS = 256       # types.cuh: threads of a g2o_eval_kernel CTA; lane pairs share a correspondence
EPSILONS = (0.01, 1e-6, 1.0)


def edge_blocks(eng):
    """mvicp_debug_edge_blocks: [E, 160] = pair matrix (12x12 row-major, src then dst) | gradient (12) | chi2 | 3 zeros."""
    lib = eng._l
    n = C.c_int32(0)
    from mv_lm_icp_b200._lib import check
    check(lib.mvicp_debug_edge_blocks(eng._ctx, None, C.c_int64(0), C.byref(n)))
    out = np.full((n.value, EOUT), np.nan)
    check(lib.mvicp_debug_edge_blocks(eng._ctx, out.ctypes.data_as(C.POINTER(C.c_double)), C.c_int64(out.size), C.byref(n)))
    return out


def gamma(k):
    return k * U / (1 - k * U)


# K_CORR, the depth of the longest chain of one correspondence in g2o_eval_kernel:
#   F0^T t0 and M01 (3-term dots) 3;  y = F1 p + t1: 4;  u = F0^T y - F0^T t0: max(4, 3) + 4 = 8;  r = u - q: 9
#   g2o_prec0: y_n (2), |y_n|^2 (3), sqrt (1), division (1) = 7, doubled for the two ways the rounding of y_n enters the
#   normalised vector (the component and the norm) = 14;  x = n x y: 16;  Omega = sum_k R_k,a d_k R_k,b: 20
#   J: the 3-term rows M01 (vx) or I (vx) from u: 11;  W = Omega J, Omega r: max(20, 11) + 3 = 23;  J^T W, J^T Omega r, r^T Omega r: 26
K_CORR = 26
K_REDUCE = 4 + EVAL_THREADS // 32      # the xor tree over lanes of equal role (16, 8, 4, 2), then the 8 warps in order


def k_depth(tl, n_tiles):
    return K_CORR + tl // (EVAL_THREADS // 2) + K_REDUCE + max(1, n_tiles)


# ---- the extended-precision reference ----------------------------------------------------------------------------------
def _skew(v):
    """[v]x for a batch [n, 3] -> [n, 3, 3]."""
    z = np.zeros(len(v), v.dtype)
    return np.stack([np.stack([z, -v[:, 2], v[:, 1]], 1), np.stack([v[:, 2], z, -v[:, 0]], 1), np.stack([-v[:, 1], v[:, 0], z], 1)], 1)


def _skew_m(v):
    z = np.zeros(len(v), v.dtype)
    return np.stack([np.stack([z, v[:, 2], v[:, 1]], 1), np.stack([v[:, 2], z, v[:, 0]], 1), np.stack([v[:, 1], v[:, 0], z], 1)], 1)


def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def _cross_m(a, b):
    return np.stack([a[:, 1] * b[:, 2] + a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] + a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] + a[:, 1] * b[:, 0]], 1)


def _inv3(F):
    """The true inverse of a 3x3 longdouble matrix (adjugate over determinant)."""
    a = np.array([[F[1, 1] * F[2, 2] - F[1, 2] * F[2, 1], F[0, 2] * F[2, 1] - F[0, 1] * F[2, 2], F[0, 1] * F[1, 2] - F[0, 2] * F[1, 1]],
                  [F[1, 2] * F[2, 0] - F[1, 0] * F[2, 2], F[0, 0] * F[2, 2] - F[0, 2] * F[2, 0], F[0, 2] * F[1, 0] - F[0, 0] * F[1, 2]],
                  [F[1, 0] * F[2, 1] - F[1, 1] * F[2, 0], F[0, 1] * F[2, 0] - F[0, 0] * F[2, 1], F[0, 0] * F[1, 1] - F[0, 1] * F[1, 0]]], LD)
    return a / (F[0] @ a[:, 0])


def _square_rounding(a):
    """fl(a * a) - a * a exactly, for fp64 a with |a| <= 2 (Dekker's TwoProduct with Veltkamp's split: every step is exact)."""
    p = a * a
    c = 134217729.0 * a
    hi = c - (c - a); lo = a - hi
    return ((hi * hi - p) + 2 * hi * lo) + lo * lo


def prec0(n, eps, mut=()):
    """(Omega [N, 3, 3], |Omega|_m, dOmega) of EdgeGICP::prec0(eps) in longdouble.  |Omega|_m: g2o_prec0's arithmetic in
    magnitudes with the normalised row 1 at |y_hat|; dOmega: what the normalisation adds, absolutely.  Row 1 as computed is
    within delta = min(2, gamma_14 |y|_m / |y|) of y_hat per component, the relative condition of normalising y (2 is the
    largest error a normalised vector can have), and Omega is linear in the rows' outer products, so dOmega = sum_k d_k (R_m
    dR + dR R_m + dR dR) over rows 0 and 1 (row 0 = n x row 1 inherits |n| delta).
    |y|_m takes y_1 = 1 - n_y^2 as the engine computes it: when fl(n_y^2) lies in [1/2, 2] the subtraction is exact (Sterbenz),
    so y_1 is off by the rounding of n_y^2 alone (computed exactly here), or by one rounding of y_1 where the product is
    contracted into an FMA; its magnitude is |rounding| / u + |y_1|.  Near n = +-e_y, where 1 - n_y^2 cancels, the plain
    magnitude 1 + n_y^2 would put the relative condition at ~2^53 and the bound of every edge carrying such a normal at O(1).
    Elsewhere y_1 keeps the magnitude 1 + n_y^2.  mut "nnT": eps I + (1 - eps) n n^T (equal only for unit normals)."""
    n1 = np.asarray(n, np.float64)[:, 1]
    sq = n1 * n1
    sterbenz = (sq >= 0.5) & (sq <= 2.0)
    rho = np.abs(_square_rounding(n1)).astype(LD)
    n = n.astype(LD); an = np.abs(n)
    if "nnT" in mut:
        Om = eps * np.eye(3, dtype=LD)[None] + (1 - eps) * np.einsum("ni,nj->nij", n, n)
        return Om, np.abs(Om), np.zeros_like(Om)
    y = np.stack([-n[:, 1] * n[:, 0], 1 - n[:, 1] * n[:, 1], -n[:, 1] * n[:, 2]], 1)
    y1_m = np.where(sterbenz, rho / LD(U) + np.abs(y[:, 1]), 1 + an[:, 1] * an[:, 1])
    y_m = np.stack([an[:, 1] * an[:, 0], y1_m, an[:, 1] * an[:, 2]], 1)
    ny = np.sqrt(np.sum(y * y, 1)); ny_m = np.sqrt(np.sum(y_m * y_m, 1))
    live = ny > 0                     # a zero vector stays zero: exactly so in fp64 too (n = (0, +-1, 0) is then exact)
    s = np.where(live, ny, 1)
    yh = np.where(live[:, None], y / s[:, None], 0)
    delta = np.where(live, np.minimum(2, gamma(14) * ny_m / s), 0)
    dy = np.broadcast_to(delta[:, None], y.shape)
    x = _cross(n, yh); x_m = _cross_m(an, np.abs(yh)); dx = _cross_m(an, dy)
    R = np.stack([x, yh, n], 1); Rm = np.stack([x_m, np.abs(yh), an], 1)      # [N, row k, column a]
    dR = np.stack([dx, dy, np.zeros_like(dy)], 1)
    d = np.array([eps, eps, 1], LD)
    Om = np.einsum("nka,k,nkb->nab", R, d, R)
    Om_m = np.einsum("nka,k,nkb->nab", Rm, d, Rm)
    dOm = np.einsum("nka,k,nkb->nab", Rm, d, dR) + np.einsum("nka,k,nkb->nab", dR, d, Rm) + np.einsum("nka,k,nkb->nab", dR, d, dR)
    return Om, Om_m, dOm


def reference_edge(Pd, Ps, p, q, n, eps, mut=()):
    """(H 12x12, g 12, chi2) of one edge's correspondences in longdouble and their magnitudes (H_m, g_m, chi2_m) in
    g2o_eval_kernel's formulation.  Pd / Ps: the dst / src 4x4 poses; n None: point-to-point.  `mut` names deliberate errors
    for the negative controls: "true_inverse" (F0^-1 for F0^T), "nnT" (the unit-normal information), "plus_I" (+I in J_dst)."""
    F0, t0 = Pd[:3, :3].astype(LD), Pd[:3, 3].astype(LD)
    F1, t1 = Ps[:3, :3].astype(LD), Ps[:3, 3].astype(LD)
    aF0, at0, aF1, at1 = np.abs(F0), np.abs(t0), np.abs(F1), np.abs(t1)
    p = p.astype(LD); q = q.astype(LD); ap, aq = np.abs(p), np.abs(q)
    N = len(p)
    F0T = _inv3(F0) if "true_inverse" in mut else F0.T
    M01 = F0T @ F1; M01_m = aF0.T @ aF1
    y = p @ F1.T + t1; y_m = ap @ aF1.T + at1
    u = y @ F0T.T - F0T @ t0; u_m = y_m @ aF0 + aF0.T @ at0
    r = u - q; r_m = u_m + aq
    if n is None:
        Om = np.broadcast_to(np.eye(3, dtype=LD), (N, 3, 3)); Om_m = Om; dOm = np.zeros_like(Om)
    else:
        Om, Om_m, dOm = prec0(n, LD(eps), mut)
    I3 = np.broadcast_to(np.eye(3, dtype=LD), (N, 3, 3))
    Jd = np.concatenate([I3 if "plus_I" in mut else -I3, 2 * _skew(u)], 2)
    Js = np.concatenate([np.broadcast_to(M01, (N, 3, 3)), -2 * np.einsum("ij,njk->nik", M01, _skew(p))], 2)
    J = np.concatenate([Js, Jd], 2)                                          # [N, 3, 12]: src then dst
    Jd_m = np.concatenate([I3, 2 * _skew_m(u_m)], 2)
    Js_m = np.concatenate([np.broadcast_to(M01_m, (N, 3, 3)), 2 * np.einsum("ij,njk->nik", M01_m, _skew_m(ap))], 2)
    J_m = np.concatenate([Js_m, Jd_m], 2)
    Or = np.einsum("nij,nj->ni", Om, r); Or_m = np.einsum("nij,nj->ni", Om_m, r_m)
    W = np.einsum("nij,njk->nik", Om, J); W_m = np.einsum("nij,njk->nik", Om_m, J_m)
    H = np.einsum("nia,nib->ab", J, W); H_m = np.einsum("nia,nib->ab", J_m, W_m)
    g = np.einsum("nia,ni->a", J, Or); g_m = np.einsum("nia,ni->a", J_m, Or_m)
    chi = np.sum(r * Or); chi_m = np.sum(r_m * Or_m)
    # what the normalisation in prec0 adds: H, g and chi2 are linear in Omega
    dW = np.einsum("nij,njk->nik", dOm, J_m)
    H_x = np.einsum("nia,nib->ab", J_m, dW); g_x = np.einsum("nia,ni->a", J_m, np.einsum("nij,nj->ni", dOm, r_m))
    chi_x = np.einsum("ni,nij,nj->", r_m, dOm, r_m)
    return H, g, chi, H_m, g_m, chi_m, H_x, g_x, chi_x


TIGHT = 1e-11   # the bound's median size relative to an edge's record: far from vacuous, yet above gamma_k of the magnitudes


def check_record(o, ref, k, what, chi=True):
    """One edge's record against reference_edge's (H, g, chi2) at gamma_k * magnitude + what the normalisation adds; chi: also
    slot 156.  The bound itself must stay tight: its median over the record is at most TIGHT of the record's scale (the largest
    diagonal entry of H for H, sqrt(that * chi2) for g -- Cauchy-Schwarz -- and chi2 for chi2), so an error of 1e-10 of that
    scale in most entries would fail.  Entries that vanish structurally (an edge whose information is rank one) do not enter a
    ratio of their own.  Returns the worst error / bound."""
    H, g, c, Hm, gm, cm, Hx, gx, cx = ref
    assert np.all(np.isfinite(o)) and not np.any(o[157:]), (what, "slots 157-159 must be zero")
    n = 157 if chi else 156
    got = o[:n].astype(LD)
    want = np.concatenate([H.ravel(), g, [c]])[:n]
    bound = (gamma(k) * np.concatenate([Hm.ravel(), gm, [cm]]) + np.concatenate([Hx.ravel(), gx, [cx]]))[:n]
    err = np.abs(got - want)
    dmax = np.max(np.abs(np.diag(H)))
    scale = np.concatenate([np.full(144, dmax), np.full(12, np.sqrt(dmax * abs(c))), [abs(c)]])[:n]
    live = scale > 0
    rel = float(np.median(bound[live] / scale[live])) if live.any() else 0.0
    assert rel <= TIGHT, (what, "the bound is too loose to test anything", rel)
    bad = np.nonzero(err > bound)[0]
    if len(bad):
        i = int(bad[np.argmax((err / np.maximum(bound, 1e-300))[bad])])
        where = f"H[{i // 12}][{i % 12}]" if i < 144 else (f"g[{i - 144}]" if i < 156 else "chi2")
        raise AssertionError(f"{what}: {len(bad)} entries out of bound; worst {where}: engine {float(got[i]):.17g} reference "
                             f"{float(want[i]):.17g} |diff| {float(err[i]):.3g} bound {float(bound[i]):.3g}")
    return float(np.max(err / np.maximum(bound, 1e-300)))


# ---- scenes -------------------------------------------------------------------------------------------------------------
def _rot(axis, th):
    a = np.asarray(axis, LD); a = a / np.sqrt(a @ a)
    K = _skew(a[None])[0]
    return (np.eye(3, dtype=LD) + np.sin(LD(th)) * K + (1 - np.cos(LD(th))) * K @ K).astype(np.float64)


AXIS = (0.3, -0.5, 0.8)
ROTATIONS = [("0", 0.0, np.eye(3)), ("1", 1.0, _rot(AXIS, 1.0)), ("pi-1e-6", math.pi - 1e-6, _rot(AXIS, math.pi - 1e-6)),
             ("pi", math.pi, np.diag([1.0, -1.0, -1.0]))]
STRONG = np.array([[1.5, 0.3, 0.0], [0.0, 0.7, 0.2], [0.1, 0.0, 1.2]])     # far from a rotation: F^-1 far from F^T


def _angle(R):
    return float(np.arccos(np.clip((np.trace(R.astype(LD)) - 1) / 2, -1, 1)))


def pose_sets(M, rng):
    """(name, kind, poses): every rotation of ROTATIONS on some frame in each of two rigid sets, frame 0 (the fixed dst of
    several edges) included; non-rigid sets where every frame, frame 0 included, is a rotation times BUMP, times
    diag(1 +- 1e-3), or times STRONG.  Asserts the property that selects each set."""
    out = []
    for shift in (0, 2):
        P = np.stack([np.eye(4)] * M)
        names = []
        for f in range(M):
            name, th, R = ROTATIONS[(f + shift) % len(ROTATIONS)]
            P[f, :3, :3] = R; P[f, :3, 3] = rng.uniform(-0.2, 0.2, 3)
            assert abs(_angle(R) - th) <= 1e-8 and np.abs(R.T @ R - np.eye(3)).max() <= 4 * U, name
            names.append(name)
        out.append(("rigid:" + ",".join(names), "rigid", P))
    for kind, S in (("bump", BUMP), ("diag", np.diag([1 + 1e-3, 1 - 1e-3, 1 + 1e-3])), ("strong", STRONG)):
        P = np.stack([np.eye(4)] * M)
        for f in range(M):
            P[f, :3, :3] = ROTATIONS[f % len(ROTATIONS)][2] @ S; P[f, :3, 3] = rng.uniform(-0.2, 0.2, 3)
            F = P[f, :3, :3]
            assert np.abs(F.T @ F - np.eye(3)).max() > 1e-5, (kind, f)
            if kind == "strong":
                assert np.abs(np.linalg.inv(F) - F.T).max() > 0.1, f
        out.append((kind, "nonrigid", P))
    return out


def shape_normals(nor, edges, corr, near_ey):
    """The dst normals the correspondences read, reshaped: scaled by 0.5 and by 2 (non-unit), exactly zero, exactly (0, +-1, 0)
    (makeRot0's zero row 1) and, with near_ey, (d, 1 - k 2^-53, d') where 1 - n_y^2 cancels.  Returns the new normals."""
    out = [None if n is None else n.copy() for n in nor]
    for (_, d), (_, sec) in zip(edges, corr):
        if not len(sec):
            continue
        n = out[d]
        n[sec[3::5]] *= 0.5
        n[sec[4::5]] *= 2.0
        n[sec[0::7]] = 0.0
        n[sec[1::11]] = [0.0, 1.0, 0.0]
        n[sec[2::13]] = [0.0, -1.0, 0.0]
        if near_ey:
            m = len(sec[5::9]); k = 1 + np.arange(m) % 4
            n[sec[5::9]] = np.stack([np.array([0.0, 2.0 ** -60, 1e-9, -3e-17])[np.arange(m) % 4], 1.0 - k * 2.0 ** -53,
                                     np.array([0.0, -2.0 ** -58, 2e-9, 0.0])[np.arange(m) % 4]], 1)
    return out


def _used_normals(nor, edges, corr):
    return np.concatenate([nor[d][sec] for (_, d), (_, sec) in zip(edges, corr) if len(sec)])


def g2o_block_scene(tl, f64=False, offset=0.0):
    """g2o_tile_scene(tl) (edges out of the fixed frame 0 with inliers on every tile's first and last slot) plus an edge of 3
    inliers ending on the last slot of frame 4's second tile: a partial warp, where the other lanes skip by __any_sync."""
    pts, nor, _, edges, corr = g2o_tile_scene(tl)
    T = tl
    edges = edges + [(4, 3)]
    corr = corr + [(np.array([2 * T - 3, 2 * T - 2, 2 * T - 1], np.int32), np.array([5, 0, T], np.int32))]
    if f64:
        pts = [p + offset + OFF_GRID for p in pts]
    return pts, nor, edges, corr


def g2o_tile_len(pts, edges, fx):
    """The g2o streaming tile: chosen from the slots of the edges whose src frame is free."""
    return tile_len(sum(len(pts[s]) for s, _ in edges if not fx[s]))


def n_tiles(pts, edges, fx, tl, e):
    s, d = edges[e]
    return 0 if (fx[s] and fx[d]) else -(-len(pts[s]) // tl)


# ---- the check -----------------------------------------------------------------------------------------------------------
def compare_g2o_blocks(eng, pts, nor, P, edges, corr, fx, cost, eps, what, tl):
    """One build at P and one trial (readout_options): slots 0-155 of every edge against the reference at P; slot 156 against
    the reference at the trial's poses when the trial was accepted.  Returns (worst ratio, accepted)."""
    o = readout_options(); o.information_eps = eps
    eng.set_poses(P, fx)
    s, chis = eng.optimize_g2o(cost, o)
    tr = eng.g2o_trace()
    assert s["calls"] == 1 and s["trials"] == 1 and len(tr) == 1 and s["evaluations"] == 2, (what, s)
    acc = bool(tr[0, 4])
    Pa = eng.get_poses()
    out = edge_blocks(eng)
    assert out.shape == (len(edges), EOUT)
    worst = 0.0
    for e, (sf, df) in enumerate(edges):
        if (fx[sf] and fx[df]) or not len(corr[e][0]):
            assert not np.any(out[e]), (what, e, "an edge without active correspondences must hold exact zeros")
            continue
        f, sec = corr[e]
        n = None if cost == COST_P2P else nor[df][sec]
        k = k_depth(tl, n_tiles(pts, edges, fx, tl, e))
        w = (what, e, (sf, df), len(f))
        worst = max(worst, check_record(out[e], reference_edge(P[df], P[sf], pts[sf][f], pts[df][sec], n, eps), k, w, chi=False))
        if acc:
            ref_a = reference_edge(Pa[df], Pa[sf], pts[sf][f], pts[df][sec], n, eps)
            bound = gamma(k) * ref_a[5] + ref_a[8]
            assert abs(LD(out[e, 156]) - ref_a[2]) <= bound, (w, "trial chi2", out[e, 156], float(ref_a[2]), float(bound))
    if acc:                           # the trace's tchi is these slots' sum
        assert abs(math.fsum(out[:, 156]) - tr[0, 2]) <= 1e-12 * tr[0, 2], (what, tr[0])
    return worst, acc


def run_g2o_block_cases(tl, mode, offset=0.0, eps_list=EPSILONS, sets=None, report=None):
    f64 = mode == "f64"
    pts, nor0, edges, corr = g2o_block_scene(tl, f64, offset)
    M = len(pts)
    fx = fixed_flags(M, (0,))
    assert g2o_tile_len(pts, edges, fx) == tl
    assert _f32_exact(np.concatenate(pts)) == (not f64)
    nor = nor0
    if mode in ("f32", "f64"):
        nor = shape_normals(nor0, edges, corr, near_ey=f64)
        used = _used_normals(nor, edges, corr)
        ln = np.linalg.norm(used, axis=1)
        assert (ln == 0).any() and (used == [0, 1, 0]).all(1).any() and (used == [0, -1, 0]).all(1).any()
        assert (np.abs(ln - 0.5) < 1e-6).any() and (np.abs(ln - 2) < 1e-6).any()
        assert all(_f32_exact(n) for n in nor) == (not f64)                       # f32: packed fp32 normal records
        if f64:
            assert ((used[:, 1] < 1) & (used[:, 1] >= 1 - 4 * U)).sum() >= 20
    eng = Engine(); eng.set_frames(pts, None if mode == "f32_no_normals" else nor); eng.set_graph(edges)
    if mode == "f32_recomputed_normals":     # g2o_eval_kernel<true, false, P2PLANE>: fp32 points, fp64 normal records
        nor, _ = eng.recompute_normals(10)
        assert not all(_f32_exact(n) for n in nor)
    upload(eng, corr)
    rng = np.random.default_rng(tl + len(mode))
    costs = [(COST_P2P, 0.01)] + ([] if mode == "f32_no_normals" else [(COST_P2PLANE, x) for x in eps_list])
    accepted = 0
    try:
        for name, kind, P in pose_sets(M, rng):
            if sets is not None and kind not in sets:
                continue
            if offset:
                P[:, :3, 3] -= P[:, :3, :3] @ np.full(3, offset)    # keep the clouds' world images near the origin
            for cost, eps in costs:
                what = (tl, mode, offset, name, cost, eps)
                wv, acc = compare_g2o_blocks(eng, pts, nor, P, edges, corr, fx, cost, eps, what, tl)
                accepted += acc
                if report is not None:
                    key = (mode, tl, "p2p" if cost == COST_P2P else f"plane eps={eps:g}", kind)
                    report[key] = max(report.get(key, 0.0), wv)
        # an edge out of a fixed frame into a free one is active; one between two fixed frames reads as zeros
        fx2 = fixed_flags(M, (0, 2))
        assert any(fx2[s] and not fx2[d] and len(corr[e][0]) for e, (s, d) in enumerate(edges))
        assert any(fx2[s] and fx2[d] and len(corr[e][0]) for e, (s, d) in enumerate(edges))
        _, _, P = pose_sets(M, rng)[0]
        if offset:
            P[:, :3, 3] -= P[:, :3, :3] @ np.full(3, offset)
        tl2 = g2o_tile_len(pts, edges, fx2)
        compare_g2o_blocks(eng, pts, nor, P, edges, corr, fx2, costs[-1][0], costs[-1][1], (tl, mode, offset, "fixed 0 2"), tl2)
    finally:
        eng.close()
    return accepted


def _print_report(report):
    for key in sorted(report):
        print("g2o blocks worst error / bound", key, "%.3g" % report[key])


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("tl", [1024, 8192])
def test_g2o_edge_blocks_match_extended_reference(tl, mode):
    report = {}
    eps_list = EPSILONS if tl == 1024 else (0.01,)     # eps changes no slot arithmetic: one value at the 8192-slot tile
    run_g2o_block_cases(tl, mode, eps_list=eps_list, report=report)
    _print_report(report)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [1e3, 1e5])
def test_g2o_edge_blocks_far_from_origin(offset):
    """fp64 clouds 1e3 m and 1e5 m from their frames' origins: the bound scales with the magnitudes, the tolerance does not."""
    report = {}
    run_g2o_block_cases(1024, "f64", offset=offset, eps_list=(0.01,), report=report)
    _print_report(report)


# ---- assembled blocks: the model the g2o suite relies on -----------------------------------------------------------------
def assemble(pts, nor, P, edges, corr, fx, cost, eps):
    """The per-edge references summed over g2o's columns (free frames that are an end of an active edge, in frame order):
    (col, H, g, H_m, g_m, H_x, g_x, number of active edges, largest inlier count); _x: what prec0's normalisation adds."""
    act = [e for e, (s, d) in enumerate(edges) if len(corr[e][0]) and not (fx[s] and fx[d])]
    touched = {v for e in act for v in edges[e]}
    col = {}
    for f in range(len(pts)):
        if f in touched and not fx[f]:
            col[f] = 6 * len(col)
    n = 6 * len(col)
    Hs = [np.zeros((n, n), LD) for _ in range(3)]      # H, H_m, H_x
    gs = [np.zeros(n, LD) for _ in range(3)]
    for e in act:
        s, d = edges[e]
        f, sec = corr[e]
        r = reference_edge(P[d], P[s], pts[s][f], pts[d][sec], None if cost == COST_P2P else nor[d][sec], eps)
        for fa, oa in ((s, 0), (d, 6)):
            if fa not in col:
                continue
            for gv, gp in zip(gs, (r[1], r[4], r[7])):
                gv[col[fa]:col[fa] + 6] += gp[oa:oa + 6]
            for fb, ob in ((s, 0), (d, 6)):
                if fb in col:
                    for Hv, Hp in zip(Hs, (r[0], r[3], r[6])):
                        Hv[col[fa]:col[fa] + 6, col[fb]:col[fb] + 6] += Hp[oa:oa + 6, ob:ob + 6]
    return col, Hs[0], gs[0], Hs[1], gs[1], Hs[2], gs[2], len(act), max(len(corr[e][0]) for e in act)


@pytest.mark.parametrize("cost", [COST_P2P, COST_P2PLANE])
def test_model_build_matches_assembled_reference(cost):
    """g2o_model.Problem.build's fp64 H and b (= -g) against the assembled references at gamma_{K_CORR + 3 N + E}: its
    einsums sum the 3 N row products of an edge's N correspondences in an order numpy picks, then the E edges."""
    pts, nor, edges, corr = g2o_block_scene(1024)
    nor = shape_normals(nor, edges, corr, near_ey=False)
    fx = fixed_flags(len(pts), (0,))
    worst = 0.0
    for name, _, P in pose_sets(len(pts), np.random.default_rng(5)):
        col, H, g, Hm, gm, Hx, gx, E, N = assemble(pts, nor, P, edges, corr, fx, cost, 0.01)
        prob = G.Problem(pts, nor, edges, corr, [bool(v) for v in fx], cost == COST_P2PLANE)
        assert prob.col == col
        Hg, bg, _ = prob.build(list(P))
        kk = gamma(K_CORR + 3 * N + E)
        for nm, got, ref, mag, extra in (("H", Hg, H, Hm, Hx), ("b", -bg, g, gm, gx)):
            err = np.abs(got.astype(LD) - ref)
            bound = kk * mag + extra
            r = err / np.maximum(bound, 1e-300)
            i = np.unravel_index(int(np.argmax(r)), r.shape)
            assert np.all(err <= bound), (name, nm, i, float(r[i]))
            worst = max(worst, float(np.max(r)))
    print("model build worst error / bound %.3g" % worst)


# ---- negative controls: the checker catches what it is there to catch ------------------------------------------------------
def test_negative_controls_exceed_the_bound():
    """Mutated references fed through check_record against the unmutated one rounded to fp64 (a stand-in for a correct engine):
    each mutation must put some entry out of the bound, on edges that carry the degenerate makeRot0 normals (exactly zero and
    exactly (0, +-1, 0)), non-unit ones and (d, 1 - k 2^-53, d') ones, where 1 - n_y^2 cancels and the normalisation's relative
    condition is largest, at every eps: the bound is not vacuous where it is loosest."""
    rng = np.random.default_rng(2)
    N = 200
    p = rng.uniform(-0.5, 0.5, (N, 3)).astype(np.float32).astype(np.float64)
    q = rng.uniform(-0.5, 0.5, (N, 3)).astype(np.float32).astype(np.float64)
    n = rng.normal(size=(N, 3)); n /= np.linalg.norm(n, axis=1, keepdims=True)
    n[3::5] *= 0.5; n[4::5] *= 2.0
    n[0::7] = 0.0; n[1::11] = [0.0, 1.0, 0.0]; n[2::13] = [0.0, -1.0, 0.0]
    m = len(n[5::9]); kk = 1 + np.arange(m) % 4
    n[5::9] = np.stack([np.array([0.0, 2.0 ** -60, 1e-9, -3e-17])[np.arange(m) % 4], 1.0 - kk * 2.0 ** -53,
                        np.array([0.0, -2.0 ** -58, 2e-9, 0.0])[np.arange(m) % 4]], 1)
    assert ((n[:, 1] < 1) & (n[:, 1] >= 1 - 4 * U)).sum() == m
    Pd, Ps = np.eye(4), np.eye(4)
    Pd[:3, :3] = _rot(AXIS, 1.0) @ BUMP; Pd[:3, 3] = [0.1, -0.2, 0.05]
    Ps[:3, :3] = _rot((0.9, 0.3, -0.3), 2.0); Ps[:3, 3] = [-0.1, 0.1, 0.2]
    k = k_depth(1024, 1)
    cases = {"dropped correspondence": None, "transposed (src, dst) block": None, "eps I + (1 - eps) n n^T": ("nnT",),
             "true inverse of a non-rigid F0": ("true_inverse",), "+I in J_dst": ("plus_I",)}
    for cost_n, eps in [(n, x) for x in EPSILONS] + [(None, 0.01)]:
        base = reference_edge(Pd, Ps, p, q, cost_n, eps)
        engine = np.zeros(EOUT)
        engine[:144] = base[0].astype(np.float64).ravel(); engine[144:156] = base[1].astype(np.float64); engine[156] = float(base[2])
        assert check_record(engine, base, k, "unmutated") <= 1.0
        for name, mut in cases.items():
            if cost_n is None and name.startswith("eps"):
                continue
            if name == "dropped correspondence":
                ref = reference_edge(Pd, Ps, p[1:], q[1:], None if cost_n is None else cost_n[1:], eps)
            elif name.startswith("transposed"):
                H = base[0].copy(); H[:6, 6:], H[6:, :6] = base[0][:6, 6:].T.copy(), base[0][6:, :6].T.copy()
                ref = (H,) + base[1:]
            else:
                ref = reference_edge(Pd, Ps, p, q, cost_n, eps, mut)
            with pytest.raises(AssertionError, match="out of bound"):
                check_record(engine, ref, k, (name, eps))


# ---- slot 156 and the first step ---------------------------------------------------------------------------------------------
def _chol_ld(A):
    n = len(A)
    L = np.zeros((n, n), LD)
    for j in range(n):
        d = A[j, j] - L[j, :j] @ L[j, :j]
        assert d > 0
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def _chol_solve_ld(L, b):
    n = len(b)
    z = np.zeros(n, LD)
    for i in range(n):
        z[i] = (b[i] - L[i, :i] @ z[:i]) / L[i, i]
    x = np.zeros(n, LD)
    for i in reversed(range(n)):
        x[i] = (z[i] - L[i + 1:, i] @ x[i + 1:]) / L[i, i]
    return x


def _oplus_ld(P, d, ortho):
    """VertexSE3::oplusImpl in longdouble: T [R(q) | t], qw = sqrt(1 - |q|^2); ortho: F <- F - F (F^T F - I) / 2 after it."""
    F, t = P[:3, :3].astype(LD), P[:3, 3].astype(LD)
    qx, qy, qz = d[3:]
    qw = np.sqrt(1 - (qx * qx + qy * qy + qz * qz))
    R = np.array([[1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qz * qw), 2 * (qx * qz + qy * qw)],
                  [2 * (qx * qy + qz * qw), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qx * qw)],
                  [2 * (qx * qz - qy * qw), 2 * (qy * qz + qx * qw), 1 - 2 * (qx * qx + qy * qy)]], LD)
    out = np.eye(4, dtype=LD)
    out[:3, :3] = F @ R; out[:3, 3] = F @ d[:3] + t
    if ortho:
        Fn = out[:3, :3]
        out[:3, :3] = Fn - Fn @ (Fn.T @ Fn - np.eye(3, dtype=LD)) / 2
    return out


def _dR_dq(q, c, h=LD(1e-7)):
    """|d R(q) / d q_c| of fromVectorMQT (qw = sqrt(1 - |q|^2)) by a central difference in longdouble: O(h^2) = 1e-14 of it."""
    e = np.zeros(3, LD); e[c] = h
    d6 = lambda v: np.concatenate([np.zeros(3, LD), v])            # noqa: E731
    return np.abs(_oplus_ld(np.eye(4), d6(q + e), False)[:3, :3] - _oplus_ld(np.eye(4), d6(q - e), False)[:3, :3]) / (2 * h)


def first_step_scene(nonrigid):
    pts, nor, poses = synthetic(4, 1500, 31, False, nonrigid)
    edges = synth.ring_edges(4, 2)
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges); eng.set_poses(poses)
    eng.correspond(0.05)
    corr = [eng.get_edge(e)[:2] for e in range(len(edges))]
    return eng, pts, nor, poses, edges, corr


def check_first_step(ortho_after, nonrigid):
    """One call, one iteration, one trial, accepted: slot 156 at the accepted poses, its sum against the trace's tchi, and the
    poses against the step solved in longdouble from the reference H and g, entry by entry.  Bound on the step, A = H +
    lambda I: the engine factors A + dA_r and solves against -g + dg_r, with |dA_r| <= gamma_{k+E} H_m + H_x (+ lambda's share
    through max H_jj) and |dg_r| <= gamma_{k+E} g_m + g_x; its Cholesky solve is backward stable, (A + dA_r + dA_c) dx' = -g +
    dg_r with |dA_c| <= gamma_{3n+1} |L| |L^T| (Higham, Thm 10.4).  So dx' - dx = A^-1 (dg_r - (dA_r + dA_c) dx') and
        |dx' - dx| <= B  for any B >= |A^-1| (|dg_r| + (|dA_r| + |dA_c|) (|dx| + B)),
    which is checked for B = 1.001 T^6(0) (a nonnegative map with T(B) <= B bounds every solution of e <= T(e)).  Through
    oplus, per frame: |dt| <= |F| |dd_t|; |dR| <= sum_c |dR/dq_c| |dq_c| (the derivative by a central difference, 1.001 for
    its error) plus the second-order 8 (sum |dq|)^2 (|d^2 R / dq^2| <= 16 for |q| < 1/2), so |dF| <= |F| |dR|; the orthonormalisation G(F) = (3 F - F F^T F) / 2 moves by at most
    (3 |dF| + |dF| |F|^T |F| + |F| |dF|^T |F| + |F| |F|^T |dF|) / 2; and the update's own rounding, gamma_40 of its
    magnitudes."""
    eng, pts, nor, poses, edges, corr = first_step_scene(nonrigid)
    if nonrigid:
        assert all(np.abs(P[:3, :3].T @ P[:3, :3] - np.eye(3)).max() > 1e-5 for P in poses[1:])
    fx = fixed_flags(len(pts), (0,))
    o = readout_options(); o.orthonormalize_after = ortho_after
    eng.set_poses(poses, fx)
    s, _ = eng.optimize_g2o(COST_P2PLANE, o)
    tr = eng.g2o_trace()
    assert s["accepted"] == 1 and len(tr) == 1 and tr[0, 4] == 1.0, (s, tr)
    Pa = eng.get_poses()
    out = edge_blocks(eng)
    tl = g2o_tile_len(pts, edges, fx)
    for e, (sf, df) in enumerate(edges):
        f, sec = corr[e]
        if not len(f):
            assert not np.any(out[e]); continue
        k = k_depth(tl, n_tiles(pts, edges, fx, tl, e))
        ref_a = reference_edge(Pa[df], Pa[sf], pts[sf][f], pts[df][sec], nor[df][sec], 0.01)
        assert abs(LD(out[e, 156]) - ref_a[2]) <= gamma(k) * ref_a[5] + ref_a[8], (e, out[e, 156], float(ref_a[2]))
    assert abs(math.fsum(out[:, 156]) - tr[0, 2]) <= 1e-12 * tr[0, 2], (math.fsum(out[:, 156]), tr[0])
    # the step
    col, H, g, Hm, gm, Hx, gx, E, _ = assemble(pts, nor, poses, edges, corr, fx, COST_P2PLANE, 0.01)
    n = len(g)
    kE = gamma(k_depth(tl, max(n_tiles(pts, edges, fx, tl, e) for e in range(len(edges)))) + E)
    tau = LD(o.tau)
    jmax = int(np.argmax(np.abs(np.diag(H))))
    lam = tau * np.abs(H[jmax, jmax])
    A = H + lam * np.eye(n, dtype=LD)
    L = _chol_ld(A)
    dx = _chol_solve_ld(L, -g)
    Ainv = np.abs(np.stack([_chol_solve_ld(L, np.eye(n, dtype=LD)[j]) for j in range(n)], 1))
    dA = kE * Hm + Hx + (tau * kE * np.max(np.diag(Hm)) + U * lam) * np.eye(n, dtype=LD) + gamma(3 * n + 1) * np.abs(L) @ np.abs(L.T)
    dg = kE * gm + gx
    T = lambda B: Ainv @ (dg + dA @ (np.abs(dx) + B))           # noqa: E731
    Bd = np.zeros(n, LD)
    for _ in range(6):
        Bd = T(Bd)
    Bd = Bd * LD(1.001)
    assert np.all(T(Bd) <= Bd), "the step's perturbation bound does not close"
    worst = top = emax = 0.0
    E3 = np.eye(3, dtype=LD)
    for f in range(len(pts)):
        if f not in col:
            assert np.array_equal(Pa[f], poses[f]), f
            continue
        c0 = col[f]
        d, dd = dx[c0:c0 + 6], Bd[c0:c0 + 6]
        assert d[3:] @ d[3:] < 0.25
        want = _oplus_ld(poses[f], d, ortho_after == 0)
        F = np.abs(poses[f][:3, :3]).astype(LD)
        inc = np.abs(_oplus_ld(np.eye(4), d, False))
        sq = np.sum(dd[3:])
        dR = sum(_dR_dq(d[3:], c) * dd[3 + c] for c in range(3)) * LD(1.001) + 8 * sq * sq
        dF = F @ dR
        dt = F @ dd[:3]
        Fo = F @ inc[:3, :3]                                          # |F R(q)|
        mag = np.zeros((4, 4), LD)
        mag[:3, :3] = Fo; mag[:3, 3] = F @ inc[:3, 3] + np.abs(poses[f][:3, 3])
        if ortho_after == 0:
            dF = (3 * dF + dF @ Fo.T @ Fo + Fo @ dF.T @ Fo + Fo @ Fo.T @ dF) / 2
            mag[:3, :3] = (3 * Fo + Fo @ Fo.T @ Fo) / 2
        bound = gamma(40) * mag
        bound[:3, :3] += dF; bound[:3, 3] += dt
        bound[3] = 0
        err = np.abs(Pa[f].astype(LD) - want)
        assert np.all(err[3] == 0), f
        r = float(np.max(err[:3] / bound[:3]))
        assert r <= 1.0, (f, r, float(np.max(err)), float(np.max(bound)))
        worst = max(worst, r); top = max(top, float(np.max(bound))); emax = max(emax, float(np.max(err)))
    print(f"first step (ortho_after {ortho_after}, nonrigid {nonrigid}): largest step bound {float(np.max(Bd)):.3g} "
          f"(|dx| up to {float(np.max(np.abs(dx))):.3g}), largest pose bound {top:.3g}, largest error {emax:.3g}, "
          f"worst error / bound {worst:.3g}")
    # the bound is set by the gradient: g = sum J^T Omega e cancels (|g| ~ g_m / 300 here), and its rounding bound
    # gamma_{k+E} g_m reaches dx through |A^-1|; still an order below the 1e-8 of the one-iteration solve tests
    assert top < 1e-9, top
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("nonrigid", [False, True])
@pytest.mark.parametrize("ortho_after", [0, 1000])
def test_first_step_and_trial_chi2(ortho_after, nonrigid):
    check_first_step(ortho_after, nonrigid)


def check_failed_factorisation_build_chi2():
    """test_failed_factorisation_is_a_rejected_trial's scene: every trial fails to factor and runs no evaluation, so slot 156 is
    the build's chi2 at the start point and sums to the trace's chi; slots 0-155 are that build's blocks."""
    rng = np.random.default_rng(17)
    dst = (rng.normal(size=(300, 3)) * 0.1).astype(np.float32).astype(np.float64)
    src = (rng.normal(size=(300, 3)) * 0.1).astype(np.float32).astype(np.float64)
    src[:40] = 0.0
    from test_gpu_lm_graphs import _rigid
    pts, edges = [dst, src], [(1, 0)]
    poses = np.stack([np.eye(4), _rigid(rng, 0.05, 0.02)])
    corr = [(np.arange(40, dtype=np.int32), rng.choice(len(dst), 40, replace=False).astype(np.int32))]
    eng = Engine(); eng.set_frames(pts, None); eng.set_graph(edges); upload(eng, corr)
    o = default_g2o_options(); o.tau = 0.0; o.max_calls = 1
    fx = np.array([1, 0], np.uint8)
    eng.set_poses(poses, fx)
    s, _ = eng.optimize_g2o(COST_P2P, o)
    tr = eng.g2o_trace()
    assert s["accepted"] == 0 and np.all(tr[:, 2] == np.inf) and s["evaluations"] == 1, (s, tr)
    assert np.array_equal(eng.get_poses(), poses)
    out = edge_blocks(eng)
    tl = g2o_tile_len(pts, edges, fx)
    ref = reference_edge(poses[0], poses[1], src[corr[0][0]], dst[corr[0][1]], None, 0.01)
    check_record(out[0], ref, k_depth(tl, n_tiles(pts, edges, fx, tl, 0)), "failed factorisation")
    assert abs(math.fsum(out[:, 156]) - tr[0, 1]) <= 1e-12 * tr[0, 1] and out[0, 156] == s["chi2_initial"], (out[0, 156], tr[0], s)
    eng.close()


@pytest.mark.gpu
def test_build_chi2_after_failed_factorisation():
    check_failed_factorisation_build_chi2()


# ---- readout state, interleaved solves, components -------------------------------------------------------------------------
def check_readout_state_and_interleaving():
    """No records before any solve or after set_graph; LM -> g2o -> LM -> g2o on one engine, each solve's records passing that
    solve's check; a call refused for its options leaves the records as they were; a g2o solve without a vertex (every frame fixed) reads as zeros although an LM solve filled the buffer."""
    import test_gpu_lm_blocks as B
    from test_gpu_lm_graphs import tile_scene
    pts, nor, edges, corr, w, _ = B.block_scene(1024)
    poses = tile_scene(1024)[2]
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges)
    with pytest.raises(MvicpError):
        edge_blocks(eng)
    for e in range(len(edges)):
        eng.set_edge(e, corr[e][0], corr[e][1], w[e])
    fx_lm = _fixed_list(len(pts), (0,))
    fx = fixed_flags(len(pts), (0,))
    tl = g2o_tile_len(pts, edges, fx)
    for kind in ("lm", "g2o", "lm", "g2o"):
        if kind == "lm":
            B.compare_blocks(eng, None, pts, nor, poses, edges, corr, w, fx_lm, PARAM_SE3, COST_P2PLANE, 0.0, 1024, ("lm", kind),
                             use_oracle=False)
        else:
            compare_g2o_blocks(eng, pts, nor, poses, edges, corr, fx, COST_P2PLANE, 0.01, ("interleaved", kind), tl)
    kept = edge_blocks(eng)
    assert np.any(kept)
    bad = readout_options(); bad.max_calls = 0
    with pytest.raises(MvicpError):                           # refused for its options: touches nothing
        eng.optimize_g2o(COST_P2PLANE, bad)
    assert np.array_equal(edge_blocks(eng), kept)
    eng.set_poses(poses, [1] * len(pts))
    s, _ = eng.optimize_g2o(COST_P2PLANE, readout_options())
    assert s["ended"] == 2 and s["trials"] == 0, s          # MVICP_G2O_END_NO_VERTICES
    out = edge_blocks(eng)
    assert out.shape == (len(edges), EOUT) and not np.any(out)
    eng.set_graph(edges)
    with pytest.raises(MvicpError):
        edge_blocks(eng)
    eng.close()


@pytest.mark.gpu
def test_readout_state_and_interleaved_solves():
    check_readout_state_and_interleaving()


def check_components(n=400):
    """Three components: {0, 1, 2} with a vertex; {3, 4}, every frame fixed (no problem); {5, 6}, whose only edge has no inlier
    (no vertex).  A joint LM evaluation fills every record first; after optimize_g2o_components the second and third components
    read as zeros and the first passes the check."""
    rng = np.random.default_rng(9)
    M = 7
    pts = [rng.uniform(-0.5, 0.5, (n, 3)).astype(np.float32).astype(np.float64) for _ in range(M)]
    nor = [rng.normal(size=(n, 3)) for _ in range(M)]
    nor = [(v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32).astype(np.float64) for v in nor]
    edges = [(1, 0), (2, 1), (0, 2), (4, 3), (3, 4), (6, 5)]
    idx = np.arange(0, n, 3, dtype=np.int32)
    corr = [(idx, rng.integers(0, n, len(idx)).astype(np.int32)) for _ in edges[:-1]] + [(np.zeros(0, np.int32),) * 2]
    w = [np.float32(0.3)] * (len(edges) - 1) + [np.float32(0)]
    P = np.stack([np.eye(4)] * M)
    for f in range(M):
        P[f, :3, :3] = ROTATIONS[f % len(ROTATIONS)][2]; P[f, :3, 3] = rng.uniform(-0.2, 0.2, 3)
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges)
    for e in range(len(edges)):
        eng.set_edge(e, corr[e][0], corr[e][1], w[e])
    assert eng.components()[1].tolist() == [0, 0, 0, 1, 1, 2, 2]
    from mv_lm_icp_b200.api import default_options
    opt = default_options(); opt.max_num_iterations = 0
    eng.set_poses(P, _fixed_list(M, (0,)))
    eng.optimize(PARAM_SE3, COST_P2PLANE, True, options=opt)
    before = edge_blocks(eng)
    assert np.any(before[3]) and np.any(before[4])          # the LM records of the second component are in the buffer
    fx = _fixed_list(M, (0, 3, 4, 5))
    eng.set_poses(P, fx)
    summ = [s for s, _ in eng.optimize_g2o_components(COST_P2PLANE, readout_options())]
    assert [s["ended"] for s in summ][1:] == [2, 2] and summ[0]["trials"] == 1, summ   # MVICP_G2O_END_NO_VERTICES
    out = edge_blocks(eng)
    assert not np.any(out[3:]) and np.all(np.isfinite(out))
    tl = g2o_tile_len(pts, edges, fx)
    for e in range(3):
        sf, df = edges[e]
        f, sec = corr[e]
        ref = reference_edge(P[df], P[sf], pts[sf][f], pts[df][sec], nor[df][sec], 0.01)
        check_record(out[e], ref, k_depth(tl, n_tiles(pts, edges, fx, tl, e)), ("components", e), chi=False)
    eng.close()


@pytest.mark.gpu
def test_readout_after_component_solve():
    check_components()
