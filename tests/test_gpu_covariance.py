"""Pose covariances of the LM problem (Engine.covariance / mvicp_covariance): C = S (S H S)^-1 S with S = diag(1 / sqrt(H_jj)),
H = J^T J at the current poses, in the tangent space of each parameterisation, per connected component.

Bar against the oracle: H from oracle.evaluate at the engine's poses, correspondences (get_edge) and weights, inverted in numpy
with the same Jacobi scaling.  Both sides carry the rounding of H (a summation of depth k per entry, entries of S H S perturbed
by about k u) through the inverse, so every entry is held to
    |C_engine - C_oracle|_ij <= c kappa(S H S) u sqrt(C_ii C_jj),   c = 4 n k,  k = 64 + E,
n unknowns, E edges: the conditioning of the problem sets the bound, not a fit.  The oracle's angle-axis Jacobian loses about
u / theta for rotation angles 0 < theta < 1 (tests/test_gpu_lm_blocks.py), so angle-axis bounds take a factor 1 / theta_min.
Each check returns the largest ratio to its bound."""
import ctypes as C

import numpy as np
import pytest

import test_gpu_components as T
import test_gpu_lm_graphs as G
from helpers import oracle_correspond, scene
from mv_lm_icp_b200 import (COST_MIXED, COST_P2P, COST_P2PLANE, COV_FIXED, COV_INDEPENDENT, COV_OK, COV_SINGULAR, PARAM_AA,
                            PARAM_QUAT, PARAM_SE3, Engine, MvicpError, synth)
from mv_lm_icp_b200.api import default_g2o_options

pytestmark = pytest.mark.gpu
U = 2.0 ** -53


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _all_pairs(M):
    return [(a, b) for a in range(M) for b in range(M)]


def _fixed_of(eng_fixed):
    fx = list(eng_fixed)
    fx[0] = 1
    return fx


def engine_problem(eng, edges, fixed):
    """(poses, correspondences, weights) of the engine's current problem: edges of a fixed src contribute nothing."""
    P = eng.get_poses()
    corr, w = [], []
    for e, (s, _) in enumerate(edges):
        if fixed[s]:
            corr.append((np.zeros(0, np.int32), np.zeros(0, np.int32))); w.append(np.float32(0)); continue
        f, sec, _, wt = eng.get_edge(e)
        corr.append((f, sec)); w.append(np.float32(wt))
    return P, corr, w


def _components(M, edges):
    """Connected component of every frame (labels only)."""
    up = list(range(M))

    def root(f):
        while up[f] != f:
            f = up[f]
        return f
    for s, d in edges:
        up[max(root(s), root(d))] = min(root(s), root(d))
    return [root(f) for f in range(M)]


def _theta_min(P):
    th = [np.arccos(np.clip((np.trace(p[:3, :3]) - 1) / 2, -1, 1)) for p in P]
    th = [t for t in th if 0 < t < 1]
    return min(th) if th else 1.0


def check_oracle(O, eng, pts, nor, edges, fixed, param, cost, robust, what=""):
    """Every (a, b) block of the engine against S (S H S)^-1 S from oracle.evaluate.  fixed: the engine's fixed flags (frame
    0 is fixed by the call in any case).  Returns the worst ratio to the bound of the module docstring."""
    M = len(pts)
    fx = _fixed_of(fixed)
    cov, st = eng.covariance(_all_pairs(M), param, cost, robust)
    P, corr, w = engine_problem(eng, edges, fx)
    nr = [None] * M if cost == COST_P2P else nor
    _, H, _ = O.evaluate(pts, nr, P, edges, corr, w, param=param, cost=cost, robust=robust, threads=8, fixed=fx)
    free = [f for f in range(M) if not fx[f]]
    col = {f: 6 * i for i, f in enumerate(free)}
    n = 6 * len(free)
    s = 1.0 / np.sqrt(np.diag(H))
    Ht = s[:, None] * H * s[None, :]
    Cref = s[:, None] * np.linalg.inv(Ht) * s[None, :]
    kappa = np.linalg.cond(Ht)
    c = 4 * n * (64 + len(edges))
    if param == PARAM_AA:
        c /= _theta_min(P)
    comp = _components(M, edges)
    worst = 0.0
    for k, (a, b) in enumerate(_all_pairs(M)):
        if fx[a] or fx[b]:
            assert st[k] == COV_FIXED and not np.any(cov[k]), (what, a, b, st[k])
            continue
        if comp[a] != comp[b]:
            assert st[k] == COV_INDEPENDENT and not np.any(cov[k]), (what, a, b, st[k])
            continue
        assert st[k] == COV_OK, (what, a, b, st[k], kappa)
        ref = Cref[col[a]:col[a] + 6, col[b]:col[b] + 6]
        da, db = np.diag(Cref)[col[a]:col[a] + 6], np.diag(Cref)[col[b]:col[b] + 6]
        bound = c * kappa * U * np.sqrt(np.outer(da, db))
        r = float(np.max(np.abs(cov[k] - ref) / bound))
        assert r <= 1.0, (what, a, b, r, kappa)
        worst = max(worst, r)
    return worst


# ---- 1. against the oracle ----------------------------------------------------------------------------------------------
def ring_engine(n_views=6, n_points=1500, rounds=3, cfg=43):
    sc = scene(n_views, n_points, cfg)
    edges = synth.ring_edges(n_views, 2)
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges); eng.set_poses(sc["poses_init"])
    for _ in range(rounds):
        eng.icp_round(0.05, PARAM_SE3, COST_P2PLANE, True)
    return eng, sc["pts"], sc["nor"], edges


def check_ring_grid(O, params=(PARAM_AA, PARAM_QUAT, PARAM_SE3), costs=(COST_P2P, COST_P2PLANE, COST_MIXED), robusts=(False, True),
                    n_points=1500):
    eng, pts, nor, edges = ring_engine(n_points=n_points)
    fixed = [1] + [0] * (len(pts) - 1)
    worst = {}
    for param in params:
        for cost in costs:
            for robust in robusts:
                worst[(param, cost, robust)] = check_oracle(O, eng, pts, nor, edges, fixed, param, cost, robust, (param, cost, robust))
    eng.close()
    return worst


def test_ring_grid_matches_oracle(oracle):
    worst = check_ring_grid(oracle)
    print("worst ratio to the bound per (param, cost, robust):", {k: round(v, 4) for k, v in worst.items()})


@pytest.mark.parametrize("mode", G.MODES)
@pytest.mark.parametrize("path", ["unit", "general"])
def test_storage_modes_and_paths(oracle, mode, path):
    eng, pts, nor, poses, edges, corr, w = G._storage_setup(oracle, mode, path)
    fx = G._fixed_list(len(pts), (0,))
    eng.set_poses(poses, fx)
    for e, (s, _) in enumerate(edges):
        if not fx[s]:
            eng.set_edge(e, corr[e][0], corr[e][1], w[e])
    worst = 0.0
    for param in ((PARAM_QUAT, PARAM_SE3) if path == "general" else (PARAM_AA, PARAM_QUAT, PARAM_SE3)):
        for cost in ([COST_P2P] if mode == "f32_no_normals" else [COST_P2P, COST_P2PLANE]):
            worst = max(worst, check_oracle(oracle, eng, pts, nor, edges, fx, param, cost, True, (mode, path, param, cost)))
    eng.close()
    print("worst ratio", worst)


def graph_engine(O, M, edges, fixed, n_points=1200, cfg=43, views=None):
    sc = scene(M, n_points, cfg)
    order = list(range(M)) if views is None else [views.index(f) for f in range(M)]
    pts, nor = [sc["pts"][v] for v in order], [sc["nor"][v] for v in order]
    poses = sc["poses_init"][order].copy()
    corr, w = G._corr_of(oracle_correspond(O, pts, poses, edges))
    fx = G._fixed_list(M, fixed)
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges); eng.set_poses(poses, fx)
    for e, (s, _) in enumerate(edges):
        if not fx[s]:
            eng.set_edge(e, corr[e][0], corr[e][1], w[e])
    return eng, pts, nor, fx


@pytest.mark.parametrize("name", G.TOPOLOGIES)
def test_topologies(oracle, name):
    M, edges, fixed = G.topology(name)
    eng, pts, nor, fx = graph_engine(oracle, M, edges, fixed, views=G.HUB_RING if name == "hub_last" else None)
    check_oracle(oracle, eng, pts, nor, edges, fx, PARAM_SE3, COST_P2PLANE, True, name)
    eng.close()


@pytest.mark.parametrize("fixed", G.FIXED_SETS[1:], ids=lambda f: "fixed" + "_".join(map(str, f)))
def test_fixed_sets(oracle, fixed):
    M, edges, _ = G.topology("ring_chord")
    eng, pts, nor, fx = graph_engine(oracle, M, edges, fixed)
    check_oracle(oracle, eng, pts, nor, edges, fx, PARAM_QUAT, COST_MIXED, True, fixed)
    eng.close()


def test_wide_component_factor_in_global_memory(oracle):
    edges = G.wide_graph(48)
    assert G.skyline_bytes(48, edges, (0,))[0] > G.SMEM_LIMIT
    eng, pts, nor, fx = graph_engine(oracle, 48, edges, (0,), n_points=600)
    check_oracle(oracle, eng, pts, nor, edges, fx, PARAM_SE3, COST_P2PLANE, True, "wide")
    eng.close()


# ---- 2. batches ---------------------------------------------------------------------------------------------------------
def _fresh_cov(c, poses, fx, param, cost, robust, mode="f32"):
    """Engine.covariance in an engine that holds only component c at the given poses and fixed flags: every local pair."""
    eng = Engine()
    T._load(eng, c.pts, c.nor, poses, fx, c.edges, lambda e: (c.corr[e][0], c.corr[e][1], c.w[e]), mode)
    out = eng.covariance(_all_pairs(c.n), param, cost, robust)
    eng.close()
    return out


def check_batch_cov(O, comps, param=PARAM_SE3, cost=COST_P2PLANE, robust=True):
    """optimize_components on the batch, then every pair of the batch: blocks within a component equal a fresh engine holding
    only that component bit for bit (same tile length and eval path), pairs across components are INDEPENDENT zeros, pairs with
    a fixed frame FIXED zeros."""
    b = T.Batch(comps)
    eng = Engine()

    def corr(e):
        k, r = b.emap[e]
        return b.comps[k].corr[r][0], b.comps[k].corr[r][1], b.comps[k].w[r]
    T._load(eng, b.pts, b.nor, b.poses, b.fx, b.edges, corr, "f32")
    eng.optimize_components(param, cost, robust)
    P = eng.get_poses()
    fx = list(b.fx)
    for k in range(len(comps)):
        fx[b.gid[k][0]] = 1               # the lowest frame of every component is now fixed
    pairs = _all_pairs(b.M)
    cov, st = eng.covariance(pairs, param, cost, robust)
    eng.close()
    comp = {g: k for k in range(len(comps)) for g in b.gid[k]}
    loc = {g: i for k in range(len(comps)) for i, g in enumerate(b.gid[k])}
    tl = G.tile_len(b.active_slots())
    general = param != PARAM_AA and T._nonrigid_poses(b.poses)
    statuses = set()
    fresh = {}
    for idx, (a, bb) in enumerate(pairs):
        statuses.add(int(st[idx]))
        if fx[a] or fx[bb]:
            assert st[idx] == COV_FIXED and not np.any(cov[idx]), (a, bb)
            continue
        if comp[a] != comp[bb]:
            assert st[idx] == COV_INDEPENDENT and not np.any(cov[idx]), (a, bb)
            continue
        k = comp[a]; c = comps[k]
        assert G.tile_len(c.active_slots()) == tl and (param != PARAM_AA and T._nonrigid_poses(c.poses)) == general
        if k not in fresh:
            fresh[k] = _fresh_cov(c, P[b.gid[k]], [fx[g] for g in b.gid[k]], param, cost, robust)
        fc, fs = fresh[k]
        j = loc[a] * c.n + loc[bb]
        assert st[idx] == fs[j], (a, bb, st[idx], fs[j])
        assert np.array_equal(_bits(cov[idx]), _bits(fc[j])), (a, bb, np.max(np.abs(cov[idx] - fc[j])))
    return statuses


def test_batch_matches_fresh_engines(oracle):
    comps = T.mixed_comps(oracle, n_points=800, wide=True)
    statuses = check_batch_cov(oracle, comps)
    # the component with a free frame without inliers is singular; others are fine
    assert statuses == {COV_OK, COV_FIXED, COV_INDEPENDENT, COV_SINGULAR}, statuses


def check_floating_component(O, n_points=800):
    """A joint graph of two components with only frame 0 fixed: the floating one is SINGULAR (NaN), the other OK with the same
    bits as when it is alone."""
    ca = T.Comp(O, 4, synth.ring_edges(4, 2), cfg=51, n_points=n_points)
    cb = T.Comp(O, 3, synth.ring_edges(3, 2), cfg=52, n_points=n_points)
    b = T.Batch([ca, cb])
    fx = [0] * b.M
    eng = Engine()

    def corr(e):
        k, r = b.emap[e]
        return b.comps[k].corr[r][0], b.comps[k].corr[r][1], b.comps[k].w[r]
    T._load(eng, b.pts, b.nor, b.poses, fx, b.edges, corr, "f32")
    assert G.tile_len(b.active_slots()) == G.tile_len(ca.active_slots())
    pairs = _all_pairs(b.M)
    cov, st = eng.covariance(pairs, PARAM_SE3, COST_P2PLANE, True)
    eng.close()
    fa, sa = _fresh_cov(ca, ca.poses, [1, 0, 0, 0], PARAM_SE3, COST_P2PLANE, True)
    for idx, (a, bb) in enumerate(pairs):
        ka = 0 if a in b.gid[0] else 1; kb = 0 if bb in b.gid[0] else 1
        if a == 0 or bb == 0:
            assert st[idx] == COV_FIXED
        elif ka != kb:
            assert st[idx] == COV_INDEPENDENT and not np.any(cov[idx])
        elif ka == 1:
            assert st[idx] == COV_SINGULAR and np.all(np.isnan(cov[idx]))
        else:
            j = b.gid[0].index(a) * 4 + b.gid[0].index(bb)
            assert st[idx] == COV_OK == sa[j]
            assert np.array_equal(_bits(cov[idx]), _bits(fa[j])), (a, bb)


def test_floating_component_is_singular(oracle):
    check_floating_component(oracle)


# ---- 3. rank -----------------------------------------------------------------------------------------------------------
def check_planar_patch(n=400, seed=3):
    """Point-to-plane on a planar patch: translation in the plane and rotation about its normal are unobservable."""
    rng = np.random.default_rng(seed)
    p = np.zeros((n, 3)); p[:, :2] = rng.uniform(-0.5, 0.5, (n, 2))
    nor = np.tile([0.0, 0.0, 1.0], (n, 1))
    q = p.copy(); q[:, 2] += rng.normal(0, 1e-3, n)
    eng = Engine(); eng.set_frames([q, p], [nor, nor]); eng.set_graph([(1, 0)]); eng.set_poses([np.eye(4), np.eye(4)])
    eng.set_edge(0, np.arange(n), np.arange(n), 0.01)
    for param in (PARAM_AA, PARAM_QUAT, PARAM_SE3):
        cov, st = eng.covariance([(1, 1)], param, COST_P2PLANE, False)
        assert st[0] == COV_SINGULAR and np.all(np.isnan(cov[0])), (param, cov[0])
        cov, st = eng.covariance([(1, 1)], param, COST_P2P, False)   # point-to-point pins the patch down
        assert st[0] == COV_OK and np.all(np.isfinite(cov[0])), param
    eng.close()


def test_planar_patch_is_singular():
    check_planar_patch()


def check_free_frame_without_inliers(n_points=600):
    sc = scene(3, n_points, 44)
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph([(1, 0), (2, 0)]); eng.set_poses(sc["poses_init"])
    eng.correspond(0.05)
    eng.set_edge(1, np.zeros(0, np.int32), np.zeros(0, np.int32), 0.0)
    cov, st = eng.covariance(None, PARAM_SE3, COST_P2PLANE, True)
    assert list(st) == [COV_FIXED, COV_SINGULAR, COV_SINGULAR], st
    assert np.all(np.isnan(cov[1:])) and not np.any(cov[0])
    eng.close()


def test_free_frame_without_inliers_is_singular():
    check_free_frame_without_inliers()


def test_frame_far_from_origin(oracle):
    """fp64 clouds 1e5 m from the origin: the rotation and translation columns of H differ by ~1e10 in scale, so the rank rule
    only holds because of the Jacobi scaling.  The frame stays OK and matches the oracle to the bound."""
    rng = np.random.default_rng(11)
    n = 2000
    base = rng.uniform(-1, 1, (n, 3)) * [1.0, 0.8, 0.3] + 1e5 + 1.0 / 3
    nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    src = base + rng.normal(0, 1e-3, (n, 3))
    pts, nor = [base, src], [nrm, nrm]
    assert not G._f32_exact(base)
    edges = [(1, 0)]
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges); eng.set_poses([np.eye(4), np.eye(4)])
    eng.set_edge(0, np.arange(n), np.arange(n), 0.01)
    worst = 0.0
    for param in (PARAM_QUAT, PARAM_SE3):
        for cost in (COST_P2P, COST_P2PLANE):
            worst = max(worst, check_oracle(oracle, eng, pts, nor, edges, [1, 0], param, cost, False, ("far", param, cost)))
    eng.close()
    print("worst ratio", worst)


# ---- 4. meaning -------------------------------------------------------------------------------------------------------
def test_covariance_predicts_the_estimation_error():
    """400 two-frame problems in one engine, angle-axis, point-to-point, no loss, dst = T_true src + N(0, sigma^2): the
    estimation errors follow N(0, sigma^2 C).  mean e^T (sigma^2 C)^-1 e ~ chi^2_6 / 400 (mean 6, standard error sqrt(12 / 400)),
    held to 4 standard errors; the sample covariance entrywise to 4 of its standard errors."""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(5)
    K, n, sigma = 400, 60, 2e-3
    p = rng.uniform(-0.5, 0.5, (n, 3)) * [1.0, 0.7, 0.4]
    Rt = Rotation.from_rotvec([0.05, -0.03, 0.02]).as_matrix(); tt = np.array([0.03, -0.02, 0.01])
    x_true = np.concatenate([Rotation.from_matrix(Rt).as_rotvec(), tt])
    pts, poses = [], []
    for k in range(K):                      # frame 2k: dst (the component's lowest frame, fixed), 2k + 1: src
        pts.append(p @ Rt.T + tt + rng.normal(0, sigma, (n, 3))); pts.append(p.copy())
        poses += [np.eye(4), np.eye(4)]
    edges = [(2 * k + 1, 2 * k) for k in range(K)]
    eng = Engine(); eng.set_frames(pts, None); eng.set_graph(edges); eng.set_poses(poses)
    idx = np.arange(n, dtype=np.int32)
    for e in range(K):
        eng.set_edge(e, idx, idx, 1.0)
    eng.optimize_components(PARAM_AA, COST_P2P, False)
    P = eng.get_poses()
    cov, st = eng.covariance([(2 * k + 1, 2 * k + 1) for k in range(K)], PARAM_AA, COST_P2P, False)
    eng.close()
    assert np.all(st == COV_OK)
    err = np.stack([np.concatenate([Rotation.from_matrix(P[2 * k + 1][:3, :3]).as_rotvec(), P[2 * k + 1][:3, 3]]) - x_true
                    for k in range(K)])
    m = np.array([err[k] @ np.linalg.solve(sigma ** 2 * cov[k], err[k]) for k in range(K)])
    assert abs(m.mean() - 6.0) <= 4 * np.sqrt(12.0 / K), m.mean()
    Sig = sigma ** 2 * cov.mean(axis=0)
    S = err.T @ err / K                     # the true mean is zero
    se = np.sqrt((np.outer(np.diag(Sig), np.diag(Sig)) + Sig ** 2) / K)
    assert np.all(np.abs(S - Sig) <= 4 * se), np.max(np.abs(S - Sig) / se)


# ---- 5. contract -------------------------------------------------------------------------------------------------------
def check_request_independence(eng, M, param=PARAM_SE3, cost=COST_P2PLANE, robust=True, seed=0):
    """Order, subsets and duplicates change no block's bits; (b, a) is (a, b)^T exactly; repeated calls are identical."""
    pairs = _all_pairs(M)
    full, st = eng.covariance(pairs, param, cost, robust)
    again, st2 = eng.covariance(pairs, param, cost, robust)
    assert np.array_equal(_bits(full), _bits(again)) and np.array_equal(st, st2)
    at = {pr: i for i, pr in enumerate(pairs)}
    for (a, b), i in at.items():
        assert np.array_equal(_bits(full[i]), _bits(full[at[(b, a)]].T)), (a, b)
    rng = np.random.default_rng(seed)
    for _ in range(3):
        sub = [pairs[i] for i in rng.integers(0, len(pairs), max(1, len(pairs) // 3))]
        sub = sub + sub[:2]                 # duplicates
        c2, s2 = eng.covariance(sub, param, cost, robust)
        for j, pr in enumerate(sub):
            assert np.array_equal(_bits(c2[j]), _bits(full[at[pr]])) and s2[j] == st[at[pr]], pr
    d, sd = eng.covariance(None, param, cost, robust)
    for f in range(M):
        assert np.array_equal(_bits(d[f]), _bits(full[at[(f, f)]])) and sd[f] == st[at[(f, f)]]
    return st


def test_request_order_subsets_duplicates():
    eng, pts, _, _ = ring_engine(n_points=1000, rounds=2)
    for param in (PARAM_AA, PARAM_QUAT, PARAM_SE3):
        st = check_request_independence(eng, len(pts), param)
        assert set(st.tolist()) == {COV_OK, COV_FIXED}
    eng.close()


def check_no_side_effects(O, n_points=800):
    """Two engines run the same sequence of solves; one also asks for covariances between them.  Every solve ends with the same
    poses and summaries bit for bit, and of the statistics only kernel_launches moves."""
    comps = [T.Comp(O, 3, synth.ring_edges(3, 2), cfg=61, n_points=n_points),
             T.Comp(O, 4, [(1, 0), (2, 1), (1, 2), (2, 0), (3, 0)], empty=(4,), cfg=62, n_points=n_points)]
    b = T.Batch(comps)

    def corr(e):
        k, r = b.emap[e]
        return b.comps[k].corr[r][0], b.comps[k].corr[r][1], b.comps[k].w[r]
    engs = [Engine(), Engine()]
    for eng in engs:
        T._load(eng, b.pts, b.nor, b.poses, b.fx, b.edges, corr, "f32")
    g2o = default_g2o_options(); g2o.max_calls = 3
    steps = [lambda e: e.optimize(PARAM_SE3, COST_P2PLANE, True),
             lambda e: e.optimize_components(PARAM_QUAT, COST_MIXED, True),
             lambda e: e.optimize_g2o(COST_P2PLANE, g2o)[0],
             lambda e: e.optimize_components(PARAM_AA, COST_P2P, False)]
    for i, step in enumerate(steps):
        before = engs[1].stats()
        for param, cost in ((PARAM_SE3, COST_P2PLANE), (PARAM_AA, COST_MIXED)):
            engs[1].covariance(None, param, cost, True)
            engs[1].covariance([(1, 2), (2, 1)], param, cost, False)
        after = engs[1].stats()
        assert after["kernel_launches"] > before["kernel_launches"]
        assert {k: v for k, v in after.items() if k != "kernel_launches"} == {k: v for k, v in before.items() if k != "kernel_launches"}
        out = [step(e) for e in engs]
        assert out[0] == out[1], (i, out)
        assert np.array_equal(_bits(engs[0].get_poses()), _bits(engs[1].get_poses())), i
    for eng in engs:
        eng.close()


def test_calls_between_solves_change_nothing(oracle):
    check_no_side_effects(oracle)


def check_errors(n_points=300):
    sc = scene(4, n_points, 31)
    eng = Engine()
    lib = eng._l
    a = np.zeros(1, np.int32); cov = np.zeros(36); st = np.zeros(1, np.int32)
    P = lambda x, t=C.c_int32: x.ctypes.data_as(C.POINTER(t))

    def raw(param=PARAM_SE3, cost=COST_P2P, n=1, fa=P(a), fb=P(a), out=P(cov, C.c_double)):
        return lib.mvicp_covariance(eng._ctx, C.c_int32(param), C.c_int32(cost), C.c_int32(1), C.c_int32(n), fa, fb, out, P(st))
    assert raw() == 4                       # no frames
    eng.set_frames(sc["pts"], None)
    assert raw() == 4                       # no graph
    eng.set_graph([(1, 0), (2, 1), (3, 2)])
    for args in (dict(param=3), dict(param=-1), dict(cost=3), dict(n=-1), dict(fa=None), dict(fb=None), dict(out=None)):
        assert raw(**args) == 1, args
    for bad in (-1, 4):
        with pytest.raises(MvicpError) as ei:
            eng.covariance([(1, bad)], PARAM_SE3, COST_P2P)
        assert ei.value.code == 1
    with pytest.raises(MvicpError) as ei:
        eng.covariance(None, PARAM_SE3, COST_P2PLANE)   # point-to-plane without normals
    assert ei.value.code == 1
    assert raw(n=0, fa=None, fb=None, out=None) == 0
    eng.close()


def test_errors():
    check_errors()
