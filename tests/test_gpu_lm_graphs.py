"""GPU parity of the LM step on every storage mode, on arbitrary pose graphs and fixed-frame sets, and at the tile boundaries of
the streaming kernels -- against the CPU oracle on identical correspondences.

Bar (as tests/test_gpu_lm.py): equal termination, iteration and successful-step counts, initial and final cost within 1e-9
relative, poses within 1e-8.  The cost at the start point (max_num_iterations = 0) is a direct readout of lm_eval_kernel /
lm_eval_general_kernel + lm_edge_kernel and is held to 1e-12 relative, against the oracle and, on the unit-quaternion path,
against an independent numpy fp64 evaluation of the reference's cost."""
import math

import numpy as np
import pytest

from helpers import oracle_correspond, pose_rel_err, scene
from mv_lm_icp_b200 import COST_MIXED, COST_P2P, COST_P2PLANE, PARAM_AA, PARAM_QUAT, PARAM_SE3, Engine, synth
from mv_lm_icp_b200.api import TERMINATION, default_options

pytestmark = pytest.mark.gpu
TIGHT_TOL = 1e-8
COST_TOL = 1e-9
READOUT_TOL = 1e-12
NUM_SMS = 132                       # types.cuh: the H100's SM count, which sizes the LM streaming tile
SMEM_LIMIT = 220 * 1024             # mvicp.cu: the factor stays in shared memory up to this many bytes (with its vectors)
PARAMS = [PARAM_AA, PARAM_QUAT, PARAM_SE3]
COSTS = [COST_P2P, COST_P2PLANE, COST_MIXED]


# ---- helpers ---------------------------------------------------------------------------------------------------------
def _f32_exact(a):
    a = np.asarray(a)
    return bool(np.array_equal(a.astype(np.float32).astype(np.float64), a))


def _options(max_iter):
    """(engine options, oracle options) with the given iteration limit; (None, None) for the defaults."""
    if max_iter is None:
        return None, None
    from oracle import oracle as O
    a, b = default_options(), O.default_options()
    a.max_num_iterations = b.max_num_iterations = max_iter
    return a, b


def _corr_of(ref):
    corr = [((r["first"], r["second"]) if r else (np.zeros(0, np.int32), np.zeros(0, np.int32))) for r in ref]
    w = [np.float32(r["weight"]) if r else np.float32(0) for r in ref]
    return corr, w


def _fixed_list(M, fixed):
    fx = [0] * M
    for f in fixed:
        fx[f] = 1
    fx[0] = 1                       # every ceresOptimizer* fixes frame 0 itself (icp-ceres.cpp:242-244)
    return fx


def compare_solve(O, eng, pts, nor, poses, edges, corr, w, param, cost, robust, fixed=(0,), max_iter=None, tag=""):
    """One solve on the engine from `poses` with the given fixed set and correspondences, the same on the oracle, held to the
    bar of the module docstring.  Only edges with a free src are uploaded (the others contribute nothing on either side).
    Returns (engine poses, engine summary, oracle poses, oracle summary)."""
    fx = _fixed_list(len(pts), fixed)
    eopt, oopt = _options(max_iter)
    eng.set_poses(poses, fx)
    for e, (s, _) in enumerate(edges):
        if not fx[s]:
            eng.set_edge(e, corr[e][0], corr[e][1], w[e])
    summ = eng.optimize(param, cost, robust, options=eopt)
    P = eng.get_poses()
    Pref, sref, _ = O.optimize(pts, nor, poses, edges, corr, w, param=param, cost=cost, robust=robust, se3_autodiff=True,
                               threads=8, fixed=fx, options=oopt)
    what = (tag, param, cost, robust, TERMINATION[summ["termination"]], summ["num_iterations"], sref["num_iterations"])
    assert summ["termination"] == sref["termination"], what
    assert summ["num_iterations"] == sref["num_iterations"], what
    assert summ["num_successful_steps"] == sref["num_successful_steps"], what
    assert abs(summ["initial_cost"] - sref["initial_cost"]) <= COST_TOL * sref["initial_cost"], what
    assert abs(summ["final_cost"] - sref["final_cost"]) <= COST_TOL * sref["final_cost"], what
    err = pose_rel_err(P, Pref)
    assert err <= TIGHT_TOL, (what, err)
    return P, summ, Pref, sref


def row_profile(M, edges, fixed):
    """First structurally non-zero column of every row of the normal matrix (mvicp.cu, mvicp_optimize): every row of a free
    frame's block starts at the lowest column of a free frame it shares an edge with (edges of a fixed src are dropped, so are
    the (s,k) blocks of a fixed dst).  Returns (rfirst, n)."""
    fx = _fixed_list(M, fixed)
    col, n = {}, 0
    for f in range(M):
        if not fx[f]:
            col[f] = n; n += 6
    rfirst = [(r // 6) * 6 for r in range(n)]
    for s, k in edges:
        if fx[s] or fx[k]:
            continue
        lo, hi = min(col[s], col[k]), max(col[s], col[k])
        for i in range(6):
            rfirst[hi + i] = min(rfirst[hi + i], lo)
    return rfirst, n


def skyline_bytes(M, edges, fixed):
    """Bytes lm_step_kernel needs for the skyline factor and its vectors: row r over columns rfirst[r]..r, the rhs row over all
    n columns, plus 3 (n + 1) doubles of vectors.  Returns (bytes, n)."""
    rfirst, n = row_profile(M, edges, fixed)
    return 8 * (sum(r - rfirst[r] + 1 for r in range(n)) + n) + 8 * 3 * (n + 1), n


def tile_len(active_slots):
    """The LM streaming tile mvicp.cu (layout_work) picks from the total of active slots."""
    tl = 8192
    while tl > 1024 and active_slots // tl < 8 * NUM_SMS:
        tl >>= 1
    return tl


# ---- 1. storage modes x unit / general path x param x cost x robust ----------------------------------------------------
MODES = ["f32", "f32_recomputed_normals", "f64", "f32_no_normals"]
OFF_GRID = np.array([1e-3 / 3, -1e-3 / 7, 1e-3 / 11])


def _nonrigid(P):
    P = P.copy(); P[:3, :3] = P[:3, :3] @ np.diag([1 + 1e-3, 1 - 7e-4, 1 + 5e-4])
    return P


def _storage_setup(O, mode, path, n_views=4, n_points=2000, cfg=61):
    """Engine and oracle inputs of one storage mode; asserts the input property that selects the mode."""
    sc = scene(n_views, n_points, cfg)
    pts = [p.copy() for p in sc["pts"]]; nor = [n.copy() for n in sc["nor"]]
    assert all(_f32_exact(p) for p in pts) and all(_f32_exact(n) for n in nor)
    if mode == "f64":
        pts = [p + OFF_GRID for p in pts]
        v = np.concatenate(pts).ravel()
        assert np.mean(v.astype(np.float32).astype(np.float64) != v) > 0.9
    eng = Engine()
    eng.set_frames(pts, None if mode == "f32_no_normals" else nor)
    if mode == "f32_recomputed_normals":
        nor, _ = eng.recompute_normals(10)
        assert not all(_f32_exact(n) for n in nor)                    # fp64 normal records from here on
        assert max(np.abs(a - b).max() for a, b in zip(nor, sc["nor"])) > 1e-3   # and not the uploaded ones
    if mode == "f32_no_normals":
        nor = [None] * n_views
    poses = sc["poses_init"].copy()
    if path == "general":
        poses[1] = _nonrigid(poses[1])
        assert np.abs(np.linalg.svd(poses[1][:3, :3])[1] - 1).max() > 1e-4
    else:
        assert all(np.abs(P[:3, :3].T @ P[:3, :3] - np.eye(3)).max() < 1e-12 for P in poses)
    edges = synth.ring_edges(n_views, 2)
    eng.set_graph(edges)
    corr, w = _corr_of(oracle_correspond(O, pts, poses, edges))
    return eng, pts, nor, poses, edges, corr, w


def _storage_cases():
    out = []
    for mode in MODES:
        for path in ("unit", "general"):
            for param in PARAMS:
                if path == "general" and param == PARAM_AA:
                    continue              # angle-axis never takes the general frame model
                out.append(pytest.param(mode, path, param, id=f"{mode}-{path}-p{param}"))
    return out


@pytest.mark.parametrize("mode,path,param", _storage_cases())
def test_storage_modes_match_oracle(oracle, mode, path, param):
    eng, pts, nor, poses, edges, corr, w = _storage_setup(oracle, mode, path)
    for cost in ([COST_P2P] if mode == "f32_no_normals" else COSTS):
        for robust in (False, True):
            compare_solve(oracle, eng, pts, nor, poses, edges, corr, w, param, cost, robust, tag=(mode, path))
    eng.close()


# ---- 2. graph topologies ---------------------------------------------------------------------------------------------
def _random_graph(seed):
    """6-14 views, 1-4 out-edges per frame (one of them to a lower frame, so that every frame is tied to frame 0), listed in
    random order."""
    rng = np.random.default_rng(seed)
    M = int(rng.integers(6, 15))
    edges = set()
    for i in range(M):
        k = int(rng.integers(1, 5))
        if i > 0:
            edges.add((i, int(rng.integers(0, i))))
        while sum(1 for s, _ in edges if s == i) < k:
            j = int(rng.integers(0, M))
            if j != i:
                edges.add((i, j))
    edges = sorted(edges)
    rng.shuffle(edges)
    return M, [tuple(map(int, e)) for e in edges], (0,)


# Frames of the hub graph in the order the scene's views lie around the ring: ring neighbours are 2-4 frame indices apart, so
# most block rows start one or more blocks to the left of their own and some at their own block.
HUB_RING = [0, 2, 4, 6, 8, 7, 5, 3, 1]


def hub_last_edges():
    ring = [(HUB_RING[i], HUB_RING[(i + d) % 9]) for i in range(9) for d in (1, -1)]
    return ring + [(i, 8) for i in range(8) if (i, 8) not in ring] + [(8, i) for i in range(1, 8) if (8, i) not in ring]


def topology(name):
    """(n_views, edges, fixed frames) of a named pose graph."""
    if name == "ring_chord":          # loop closure across the ring, both directions
        return 8, synth.ring_edges(8, 2) + [(2, 6), (6, 2)], (0,)
    if name == "hub_last":            # the last frame sees every other one: one wide block row
        return 9, hub_last_edges(), (0,)
    if name.startswith("random"):
        return _random_graph(int(name[6:]))
    if name == "two_components":      # two rings, each tied down by its own fixed frame
        ring = lambda a, m: [(a + i, a + (i + 1) % m) for i in range(m)] + [(a + (i + 1) % m, a + i) for i in range(m)]
        return 10, ring(0, 5) + ring(5, 5), (0, 5)
    if name == "dst_only":            # frames 3 and 6 are never a src
        return 7, [(s, d) for s, d in synth.ring_edges(7, 2) if s not in (3, 6)], (0,)
    if name == "dst_fixed":           # edges into a fixed frame in the middle of the column order
        return 8, synth.ring_edges(8, 2) + [(1, 4), (7, 4)], (0, 4)
    raise KeyError(name)


TOPOLOGIES = ["ring_chord", "hub_last", "random1", "random2", "random3", "two_components", "dst_only", "dst_fixed"]


def run_graph(O, M, edges, fixed, n_points=1500, cfg=43, rounds=2, param=PARAM_SE3, cost=COST_P2PLANE, robust=True, views=None):
    """Consecutive solves on one engine, each from the oracle's previous poses with fresh oracle correspondences.  Frame f is
    the scene's view views[f] (default: view f), and the scene's views lie in that order around a ring."""
    sc = scene(M, n_points, cfg)
    order = list(range(M)) if views is None else [views.index(f) for f in range(M)]
    pts, nor = [sc["pts"][v] for v in order], [sc["nor"][v] for v in order]
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges)
    poses = sc["poses_init"][order].copy()
    for rnd in range(rounds):
        corr, w = _corr_of(oracle_correspond(O, pts, poses, edges))
        _, _, poses, _ = compare_solve(O, eng, pts, nor, poses, edges, corr, w, param, cost, robust, fixed=fixed, tag=(M, rnd))
    eng.close()


@pytest.mark.parametrize("name", TOPOLOGIES)
def test_graph_topologies_match_oracle(oracle, name):
    M, edges, fixed = topology(name)
    rfirst, n = row_profile(M, edges, fixed)
    starts = [rfirst[r] // 6 for r in range(0, n, 6)]     # first block column of every block row
    if name == "hub_last":            # one wide block row at the end; rows before it that do not reach the previous block
        assert starts[-1] == 0 and any(starts[b] == b for b in range(1, len(starts) - 1)), starts
    if name == "ring_chord":          # the chord's row reaches four blocks back
        assert starts[5] == 1, starts
    if name.startswith("random"):
        assert edges != sorted(edges)
    run_graph(oracle, M, edges, fixed, views=HUB_RING if name == "hub_last" else None)


def wide_graph(M):
    """Ring plus an edge from every frame to frame 1, the first free frame: every row's profile starts at column 0."""
    return synth.ring_edges(M, 2) + [(i, 1) for i in range(2, M) if (i, 1) not in synth.ring_edges(M, 2)]


@pytest.mark.parametrize("n_views,over", [(36, False), (48, True)])
def test_wide_graph_factor_in_global_memory(oracle, n_views, over):
    """The skyline factor leaves shared memory (lm_step_kernel then keeps it in global memory) when the row profiles are
    wide, whatever the view count: 48 views with a hub on the first free frame need ~320 KiB, 36 views ~180 KiB."""
    edges = wide_graph(n_views)
    need, n = skyline_bytes(n_views, edges, (0,))
    assert (need > SMEM_LIMIT) == over, need
    assert skyline_bytes(40, synth.ring_edges(40, 2), (0,))[0] < SMEM_LIMIT     # a plain ring of 40 views stays inside
    run_graph(oracle, n_views, edges, (0,), rounds=1)


# ---- 3. fixed-frame sets ---------------------------------------------------------------------------------------------
FIXED_SETS = [(0,), (0, 4), (0, 7), (0, 2, 5), (0, 1, 2, 4, 5, 6, 7)]


@pytest.mark.parametrize("fixed", FIXED_SETS, ids=lambda f: "fixed" + "_".join(map(str, f)))
def test_fixed_sets_match_oracle(oracle, fixed):
    M, edges, _ = topology("ring_chord")
    run_graph(oracle, M, edges, fixed, rounds=1, param=PARAM_QUAT, cost=COST_MIXED)


def test_all_frames_fixed_leaves_poses_unchanged(oracle):
    M, edges, _ = topology("ring_chord")
    sc = scene(M, 1500, 43)
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges)
    eng.set_poses(sc["poses_init"], [1] * M)
    s = eng.optimize(PARAM_SE3, COST_P2PLANE, True)
    assert TERMINATION[s["termination"]] == "GRADIENT_TOLERANCE" and s["num_iterations"] == 0
    P = eng.get_poses()
    assert np.array_equal(P.view(np.uint64), np.asarray(sc["poses_init"]).view(np.uint64))
    corr, w = _corr_of(oracle_correspond(oracle, sc["pts"], sc["poses_init"], edges))
    Pref, _, _ = oracle.optimize(sc["pts"], sc["nor"], sc["poses_init"], edges, corr, w, fixed=[1] * M, threads=8)
    assert pose_rel_err(P, Pref) <= 1e-14          # the oracle only passes them through the parameter round trip
    eng.close()


def test_switching_fixed_sets_between_solves(oracle):
    """One engine, the fixed set changed before every solve: the cached gather lists and envelope are rebuilt each time."""
    M, edges, _ = topology("ring_chord")
    sc = scene(M, 1500, 43)
    poses = sc["poses_init"]
    corr, w = _corr_of(oracle_correspond(oracle, sc["pts"], poses, edges))
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges)
    for fixed in [(0,), (0, 4), (0, 2, 5), (0,), (0, 7), (0, 4)]:
        compare_solve(oracle, eng, sc["pts"], sc["nor"], poses, edges, corr, w, PARAM_SE3, COST_P2PLANE, True, fixed=fixed,
                      tag=fixed)
    eng.close()


# ---- 4. tile boundaries and the cost readout -------------------------------------------------------------------------
def _unit(rng, n):
    v = rng.normal(size=(n, 3)); return v / np.linalg.norm(v, axis=1, keepdims=True)


def _rigid(rng, s_rot, s_tra):
    w = rng.normal(0, s_rot, 3); th = np.linalg.norm(w); k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    P = np.eye(4); P[:3, :3] = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K; P[:3, 3] = rng.normal(0, s_tra, 3)
    return P


def tile_scene(tl, seed=7):
    """Random clouds and hand-set correspondences around the tiles of length `tl`: src clouds of tl-1, tl, tl+1 and 2 tl+1
    points; inlier counts 0, 1, 2, 3, 255, 256, 257, tl-1 and tl+1; inliers on the first and last slot of every tile; a
    filler frame whose edges bring the total of active slots to the range that selects `tl`."""
    rng = np.random.default_rng(seed + tl)
    filler = {1024: (0, 0), 2048: (1_100_000, 2), 4096: (1_100_000, 4), 8192: (2_200_000, 4)}[tl]
    sizes = [3001, tl - 1, tl, tl + 1, 2 * tl + 1] + ([filler[0]] if filler[1] else [])
    pts = [rng.uniform(-0.5, 0.5, (n, 3)).astype(np.float32).astype(np.float64) for n in sizes]
    nor = [_unit(rng, n).astype(np.float32).astype(np.float64) for n in sizes]
    poses = np.stack([np.eye(4)] + [_rigid(rng, 0.05, 0.02) for _ in sizes[1:]])
    T = tl
    bounds = lambda n: sorted({k for t in range(0, n, T) for k in (t, min(t + T, n) - 1)})

    def pick(n, count, must=()):
        must = [k for k in must if k < n][:count]
        rest = np.setdiff1d(np.arange(n), must)
        return np.sort(np.concatenate([np.asarray(must, int), rng.choice(rest, count - len(must), replace=False)])).astype(np.int32)

    spec = [  # (src, dst, inlier slots)
        (1, 0, np.arange(T - 1, dtype=np.int32)),               # tl - 1 inliers: every slot of a cloud one short of a tile
        (2, 0, np.array([T - 1], np.int32)),                    # 1 inlier, on the last slot of the only tile
        (3, 0, np.array([T - 1, T], np.int32)),                 # 2 inliers straddling the tile boundary
        (4, 0, pick(2 * T + 1, T + 1, bounds(2 * T + 1))),      # tl + 1, on every tile's first and last slot
        (4, 1, np.array([0, T, 2 * T], np.int32)),              # 3: first slot of each of three tiles
        (3, 2, pick(T + 1, 255, bounds(T + 1))),
        (2, 4, pick(T, 256, bounds(T))),
        (1, 3, pick(T - 1, 257, bounds(T - 1))),
        (2, 3, np.zeros(0, np.int32)),                          # no inlier, weight 0
    ]
    if filler[1]:
        for j in range(filler[1]):
            spec.append((5, j, pick(filler[0], 1000, bounds(filler[0]))))
    edges = [(s, d) for s, d, _ in spec]
    corr, w = [], []
    for s, d, first in spec:
        corr.append((first, rng.integers(0, sizes[d], len(first)).astype(np.int32)))
        w.append(np.float32(rng.uniform(0.1, 0.4)) if len(first) else np.float32(0))
    active = sum(sizes[s] for s, _ in edges)
    return pts, nor, poses, edges, corr, w, active


def numpy_cost(pts, nor, poses, edges, corr, w, cost, robust):
    """The reference's cost in fp64 from the 4x4 poses, world frame: 1/2 sum |r|^2, or with SoftLOneLoss(a) b (sqrt(1 + s/b)
    - 1), b = a^2, per residual block; point-to-point and point-to-plane (dst normal) blocks, summed with math.fsum."""
    terms = []
    for e, (s, d) in enumerate(edges):
        if s == 0 or not len(corr[e][0]):
            continue
        Ps, Pd = poses[s], poses[d]
        x = pts[s][corr[e][0]] @ Ps[:3, :3].T + Ps[:3, 3]
        y = pts[d][corr[e][1]] @ Pd[:3, :3].T + Pd[:3, 3]
        dd = x - y
        sq = []
        if cost != COST_P2PLANE:
            sq.append(np.sum(dd * dd, axis=1))
        if cost != COST_P2P:
            sq.append(np.sum(dd * (nor[d][corr[e][1]] @ Pd[:3, :3].T), axis=1) ** 2)
        b = float(w[e]) ** 2
        for q in sq:
            terms.extend((b * (np.sqrt(1.0 + q / b) - 1.0)) if robust else 0.5 * q)
    return math.fsum(terms)


def check_tile_readout(O, tl, modes=MODES, paths=("unit", "general"), params=PARAMS, costs=COSTS, robusts=(False, True)):
    pts0, nor0, poses0, edges, corr, w, active = tile_scene(tl)
    assert tile_len(active) == tl, (active, tile_len(active))
    for mode in modes:
        pts = [p + OFF_GRID for p in pts0] if mode == "f64" else pts0
        assert _f32_exact(np.concatenate(pts)) == (mode != "f64")
        eng = Engine(); eng.set_frames(pts, None if mode == "f32_no_normals" else nor0); eng.set_graph(edges)
        nor = nor0
        if mode == "f32_recomputed_normals":
            nor, _ = eng.recompute_normals(10)
            assert not all(_f32_exact(n) for n in nor)
        if mode == "f32_no_normals":
            nor = [None] * len(pts)
        eopt, oopt = _options(0)
        for path in paths:
            poses = poses0.copy()
            if path == "general":
                poses[1] = _nonrigid(poses[1])
            for param in params:
                if path == "general" and param == PARAM_AA:
                    continue
                for cost in ([COST_P2P] if mode == "f32_no_normals" else costs):
                    for robust in robusts:
                        what = (tl, mode, path, param, cost, robust)
                        eng.set_poses(poses, _fixed_list(len(pts), (0,)))
                        for e in range(len(edges)):
                            eng.set_edge(e, corr[e][0], corr[e][1], w[e])
                        s = eng.optimize(param, cost, robust, options=eopt)
                        assert TERMINATION[s["termination"]] == "MAX_ITERATIONS" and np.isfinite(s["initial_cost"]), (what, s)
                        c_orc, _, _ = O.evaluate(pts, nor, poses, edges, corr, w, param=param, cost=cost, robust=robust,
                                                 threads=8, want_jac=False)
                        assert abs(s["initial_cost"] - c_orc) <= READOUT_TOL * c_orc, (what, s["initial_cost"], c_orc)
                        if path == "unit":
                            c_np = numpy_cost(pts, nor, poses, edges, corr, w, cost, robust)
                            assert abs(s["initial_cost"] - c_np) <= READOUT_TOL * c_np, (what, s["initial_cost"], c_np)
        # one full iteration: the normal matrix and gradient behind the first step
        cost = COST_P2P if mode == "f32_no_normals" else COST_MIXED
        compare_solve(O, eng, pts, nor, poses0, edges, corr, w, PARAM_SE3, cost, True, max_iter=1, tag=(tl, mode))
        eng.close()


@pytest.mark.parametrize("tl", [1024, 2048, 4096, 8192])
def test_tile_boundaries_cost_readout(oracle, tl):
    check_tile_readout(oracle, tl)


def test_zero_inlier_edge_with_zero_weight_adds_nothing(oracle):
    """An edge without inliers has weight 0; under the robust loss b = 0 must not turn into a NaN: the cost with it equals the
    cost without it (up to the association of the edge sums, which shifts with the edge indices)."""
    pts, nor, poses, edges, corr, w, _ = tile_scene(1024)
    eopt, _ = _options(0)
    out = []
    for drop in (False, True):
        E = [e for e in range(len(edges)) if not (drop and len(corr[e][0]) == 0)]
        eng = Engine(); eng.set_frames(pts, nor); eng.set_graph([edges[e] for e in E]); eng.set_poses(poses)
        for i, e in enumerate(E):
            eng.set_edge(i, corr[e][0], corr[e][1], w[e])
        out.append(eng.optimize(PARAM_SE3, COST_MIXED, True, options=eopt)["initial_cost"])
        eng.close()
    assert np.isfinite(out[0]) and abs(out[0] - out[1]) <= READOUT_TOL * out[1], out


# ---- 5. a free frame without residuals -------------------------------------------------------------------------------
def test_free_frame_without_residuals_counts_in_x_norm(oracle):
    """A free frame that no correspondence touches (here: its only edge has no inliers) keeps its column; its step is exactly
    zero, but its parameters enter x_norm in the parameter-tolerance test |dx| <= tol (|x| + tol).  The reference's
    quaternion and SE3 solvers cannot run this problem (Ceres rejects SetParameterization on a block that no residual
    added) and its angle-axis solver leaves the block out; the engine and the oracle keep it (DESIGN section 2).  Placed
    1e5 m away, the frame makes the tolerance 1e5 times looser, which ends the solve early: the engine must match the
    oracle with the frame, and the oracle's own run without it must differ."""
    sc = scene(4, 2000, 61)
    pts, nor = list(sc["pts"]), list(sc["nor"])
    poses = sc["poses_init"].copy()
    far = poses[1].copy(); far[:3, 3] += [1e5, -2e5, 5e4]
    edges = [(1, 0), (2, 1), (1, 2), (2, 0)]
    corr, w = _corr_of(oracle_correspond(oracle, pts[:3], poses, edges))
    pts4, nor4, poses4 = pts[:3] + [pts[3]], nor[:3] + [nor[3]], np.concatenate([poses[:3], far[None]])
    edges4 = edges + [(3, 0)]
    corr4, w4 = corr + [(np.zeros(0, np.int32), np.zeros(0, np.int32))], w + [np.float32(0)]
    for param in PARAMS:
        eng = Engine(); eng.set_frames(pts4, nor4); eng.set_graph(edges4)
        P, s, Pref, sref = compare_solve(oracle, eng, pts4, nor4, poses4, edges4, corr4, w4, param, COST_P2PLANE, True)
        eng.close()
        assert pose_rel_err(P[:3], Pref[:3]) <= TIGHT_TOL     # the far frame's 1e5 would hide their differences in the bar
        _, s3, _ = oracle.optimize(pts[:3], nor[:3], poses[:3], edges, corr, w, param=param, cost=COST_P2PLANE, robust=True,
                                   threads=8)
        assert TERMINATION[s["termination"]] == "PARAMETER_TOLERANCE", (param, s)
        assert (s3["termination"], s3["num_iterations"]) != (sref["termination"], sref["num_iterations"]), (param, s3, sref)
