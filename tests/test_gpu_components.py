"""One LM problem per connected component (Engine.optimize_components / mvicp_optimize_components).

Contract: every component ends exactly as Engine.optimize ends in a fresh engine that holds only that component (its frames in
ascending order, its edges in graph order, the same fixed flags, options and correspondences) -- poses and every summary field
bit for bit -- as long as the settings the batch shares are the same there: the streaming tile length, the unit / general
eval path and the storage mode.  Those preconditions are asserted, and each component is also held to the oracle bar of
tests/test_gpu_lm_graphs.py.  On a connected graph the call equals Engine.optimize."""
import numpy as np
import pytest

import test_gpu_lm_graphs as G
from helpers import oracle_correspond, pose_rel_err, scene
from mv_lm_icp_b200 import COST_MIXED, COST_P2P, COST_P2PLANE, PARAM_AA, PARAM_QUAT, PARAM_SE3, Engine, MvicpError, synth
from mv_lm_icp_b200.api import TERMINATION, default_options

pytestmark = pytest.mark.gpu
NO_UNKNOWNS = {"termination": 1, "num_iterations": 0, "num_successful_steps": 0, "num_evaluations": 0, "num_linear_solves": 0,
               "initial_cost": 0.0, "final_cost": 0.0}   # mvicp_optimize's summary when nothing is free (GRADIENT_TOLERANCE)


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _nonrigid_poses(poses):
    return any(np.abs(np.linalg.svd(P[:3, :3])[1] - 1).max() > 1e-9 for P in poses)


# ---- one component and a batch of them ---------------------------------------------------------------------------------
class Comp:
    """One component: n_views frames of its own scene, local edges (graph order), user-fixed local frames (local frame 0 is
    fixed in any case), the oracle's correspondences at its poses; edges listed in `empty` get no inlier and weight 0."""

    def __init__(self, O, n_views, edges, fixed=(), n_points=1200, cfg=43, start="init", nonrigid=False, empty=(), mode="f32"):
        sc = scene(n_views, n_points, cfg)
        self.pts = [p + G.OFF_GRID for p in sc["pts"]] if mode == "f64" else [p.copy() for p in sc["pts"]]
        self.nor = [n.copy() for n in sc["nor"]]
        self.poses = (sc["poses_gt"] if start == "gt" else sc["poses_init"]).copy()
        if nonrigid and n_views > 1:
            self.poses[1] = G._nonrigid(self.poses[1])
        self.n, self.edges = n_views, list(edges)
        self.fx = G._fixed_list(n_views, fixed)
        self.free = not all(self.fx)
        if self.edges:
            self.corr, self.w = G._corr_of(oracle_correspond(O, self.pts, self.poses, self.edges))
        else:
            self.corr, self.w = [], []
        for e in empty:
            self.corr[e] = (np.zeros(0, np.int32), np.zeros(0, np.int32)); self.w[e] = np.float32(0)
        if start == "solved":             # start at the oracle's solution for these correspondences: a solve that stops at once
            self.poses, _, _ = O.optimize(self.pts, self.nor, self.poses, self.edges, self.corr, self.w, threads=8, fixed=self.fx)

    def active_slots(self):
        return sum(len(self.pts[s]) for s, _ in self.edges if not self.fx[s])


class Batch:
    """The components in one engine, frames and edges interleaved round robin: component k owns frames k, k + K, ... (as far
    as it has frames), so its frames are spread over the index range but stay in ascending order, and it is component k."""

    def __init__(self, comps):
        self.comps = comps
        self.gid = [[None] * c.n for c in comps]
        M = 0
        for r in range(max(c.n for c in comps)):
            for k, c in enumerate(comps):
                if r < c.n:
                    self.gid[k][r] = M; M += 1
        self.M = M
        self.edges, self.emap = [], []
        for r in range(max(len(c.edges) for c in comps)):
            for k, c in enumerate(comps):
                if r < len(c.edges):
                    s, d = c.edges[r]
                    self.edges.append((self.gid[k][s], self.gid[k][d])); self.emap.append((k, r))
        self.pts, self.nor = [None] * M, [None] * M
        self.poses = np.zeros((M, 4, 4)); self.fx = [0] * M
        for k, c in enumerate(comps):
            for i, g in enumerate(self.gid[k]):
                self.pts[g], self.nor[g], self.poses[g], self.fx[g] = c.pts[i], c.nor[i], c.poses[i], c.fx[i]

    def active_slots(self):
        return sum(c.active_slots() for c in self.comps)


def _load(eng, pts, nor, poses, fx, edges, corr_of_edge, mode):
    """Frames, graph, poses, fixed flags and the correspondences of every edge with a free src into `eng`; returns the
    normals the solve uses (recomputed ones in that mode, None without normals)."""
    eng.set_frames(pts, None if mode == "f32_no_normals" else nor)
    out = nor
    if mode == "f32_recomputed_normals":
        out, _ = eng.recompute_normals(10)
    if mode == "f32_no_normals":
        out = [None] * len(pts)
    eng.set_graph(edges)
    eng.set_poses(poses, fx)
    for e, (s, _) in enumerate(edges):
        if not fx[s]:
            first, second, w = corr_of_edge(e)
            eng.set_edge(e, first, second, w)
    return out


def solve_fresh(c, param, cost, robust, opts, mode="f32"):
    """Engine.optimize in an engine that holds only component c: (poses, summary, normals used)."""
    eng = Engine()
    nor = _load(eng, c.pts, c.nor, c.poses, c.fx, c.edges, lambda e: (c.corr[e][0], c.corr[e][1], c.w[e]), mode)
    s = eng.optimize(param, cost, robust, options=opts)
    P = eng.get_poses()
    eng.close()
    return P, s, nor


def solve_batch(b, param, cost, robust, opts, mode="f32"):
    """Engine.optimize_components on the batch: (poses, summaries, normals used); checks the component numbering."""
    eng = Engine()

    def corr(e):
        k, r = b.emap[e]
        return b.comps[k].corr[r][0], b.comps[k].corr[r][1], b.comps[k].w[r]
    nor = _load(eng, b.pts, b.nor, b.poses, b.fx, b.edges, corr, mode)
    n, comp_of = eng.components()
    assert n == len(b.comps)
    for k in range(n):
        assert all(comp_of[g] == k for g in b.gid[k])
    summ = eng.optimize_components(param, cost, robust, options=opts)
    P = eng.get_poses()
    eng.close()
    return P, summ, nor


def check_batch(O, comps, param=PARAM_SE3, cost=COST_P2PLANE, robust=True, max_iter=None, mode="f32", oracle_bar=True):
    """The batch against a fresh engine per component (bit for bit) and against the oracle (the bar of test_gpu_lm_graphs)."""
    b = Batch(comps)
    eopt, oopt = G._options(max_iter)
    tl = G.tile_len(b.active_slots())
    P, summ, nor = solve_batch(b, param, cost, robust, eopt, mode)
    general = param != PARAM_AA and _nonrigid_poses(b.poses)
    out = []
    for k, c in enumerate(comps):
        Pk, sk = P[b.gid[k]], summ[k]
        what = (k, c.n, param, cost, robust, mode, TERMINATION[sk["termination"]], sk["num_iterations"])
        if not c.free:                    # nothing to solve: poses pass through, the summary of a problem without unknowns
            assert np.array_equal(_bits(Pk), _bits(c.poses)), what
            assert sk == NO_UNKNOWNS, (what, sk)
            out.append(sk)
            continue
        # preconditions of the bit-for-bit contract: the settings the batch shares are this component's own
        assert G.tile_len(c.active_slots()) == tl, (what, c.active_slots(), b.active_slots())
        assert (param != PARAM_AA and _nonrigid_poses(c.poses)) == general, what
        Pf, sf, _ = solve_fresh(c, param, cost, robust, eopt, mode)
        assert sk == sf, (what, sk, sf)
        assert np.array_equal(_bits(Pk), _bits(Pf)), (what, pose_rel_err(Pk, Pf))
        if oracle_bar:
            nk = [nor[g] for g in b.gid[k]]
            Pref, sref, _ = O.optimize(c.pts, nk, c.poses, c.edges, c.corr, c.w, param=param, cost=cost, robust=robust,
                                       se3_autodiff=True, threads=8, fixed=c.fx, options=oopt)
            assert sk["termination"] == sref["termination"], (what, sref)
            assert sk["num_iterations"] == sref["num_iterations"], (what, sref)
            assert sk["num_successful_steps"] == sref["num_successful_steps"], (what, sref)
            assert abs(sk["initial_cost"] - sref["initial_cost"]) <= G.COST_TOL * sref["initial_cost"], (what, sref)
            assert abs(sk["final_cost"] - sref["final_cost"]) <= G.COST_TOL * sref["final_cost"], (what, sref)
            assert pose_rel_err(Pk, Pref) <= G.TIGHT_TOL, what
        out.append(sk)
    return out


# ---- 1. connected graphs: the call is mvicp_optimize ---------------------------------------------------------------------
CONNECTED = [t for t in G.TOPOLOGIES if t != "two_components"]


def check_connected(O, name, params=G.PARAMS, costs=G.COSTS, robusts=(False, True), paths=("unit", "general"), n_points=1500):
    M, edges, fixed = G.topology(name)
    sc = scene(M, n_points, 43)
    views = G.HUB_RING if name == "hub_last" else list(range(M))
    order = [views.index(f) for f in range(M)]
    pts, nor = [sc["pts"][v] for v in order], [sc["nor"][v] for v in order]
    poses0 = sc["poses_init"][order].copy()
    corr, w = G._corr_of(oracle_correspond(O, pts, poses0, edges))
    fx = G._fixed_list(M, fixed)
    engs = [Engine(), Engine()]
    for eng in engs:
        eng.set_frames(pts, nor); eng.set_graph(edges)
    assert engs[1].components()[0] == 1
    for path in paths:
        poses = poses0.copy()
        if path == "general":
            poses[1] = G._nonrigid(poses[1])
        for param in params:
            if path == "general" and param == PARAM_AA:
                continue
            for cost in costs:
                for robust in robusts:
                    out = []
                    for i, eng in enumerate(engs):
                        eng.set_poses(poses, fx)
                        for e, (s, _) in enumerate(edges):
                            if not fx[s]:
                                eng.set_edge(e, corr[e][0], corr[e][1], w[e])
                        s = eng.optimize(param, cost, robust) if i == 0 else eng.optimize_components(param, cost, robust)[0]
                        out.append((eng.get_poses(), s))
                    what = (name, path, param, cost, robust)
                    assert out[0][1] == out[1][1], (what, out[0][1], out[1][1])
                    assert np.array_equal(_bits(out[0][0]), _bits(out[1][0])), what
    for eng in engs:
        eng.close()


@pytest.mark.parametrize("name", CONNECTED)
def test_connected_graph_equals_optimize(oracle, name):
    check_connected(oracle, name)


# ---- 2. batches ------------------------------------------------------------------------------------------------------------
def mixed_comps(O, n_points=1200, nonrigid=False, mode="f32", wide=True):
    """Two-view pairs, a ring with chords, a ring with a user-fixed frame that is not its lowest, an all-fixed ring, an
    isolated frame, a component with a free frame without inliers and (wide) a component whose factor needs global memory."""
    kw = dict(n_points=n_points, nonrigid=nonrigid, mode=mode)
    comps = [
        Comp(O, 2, [(1, 0), (0, 1)], cfg=11, **kw),
        Comp(O, 6, synth.ring_edges(6, 2) + [(1, 4), (4, 1)], cfg=12, **kw),
        Comp(O, 2, [(0, 1), (1, 0)], cfg=13, **kw),
        Comp(O, 5, synth.ring_edges(5, 2), fixed=(2,), cfg=14, **kw),
        Comp(O, 3, synth.ring_edges(3, 1), fixed=(0, 1, 2), cfg=15, **kw),
        Comp(O, 1, [], cfg=16, **kw),
        Comp(O, 4, [(1, 0), (2, 1), (1, 2), (2, 0), (3, 0)], empty=(4,), cfg=17, **kw),
    ]
    if wide:
        need, _ = G.skyline_bytes(48, G.wide_graph(48), (0,))
        assert need > G.SMEM_LIMIT and G.skyline_bytes(6, comps[1].edges, (0,))[0] < G.SMEM_LIMIT
        comps.append(Comp(O, 48, G.wide_graph(48), cfg=18, n_points=600, nonrigid=nonrigid, mode=mode))
    return comps


@pytest.mark.parametrize("param,cost,robust", [(PARAM_SE3, COST_P2PLANE, True), (PARAM_QUAT, COST_MIXED, False),
                                               (PARAM_AA, COST_P2P, True)])
@pytest.mark.parametrize("path", ["unit", "general"])
def test_batch_matches_fresh_engines_and_oracle(oracle, param, cost, robust, path):
    if path == "general" and param == PARAM_AA:
        pytest.skip("angle-axis never takes the general frame model")
    comps = mixed_comps(oracle, nonrigid=path == "general")
    sums = check_batch(oracle, comps, param, cost, robust)
    assert len({(s["termination"], s["num_iterations"]) for s in sums}) > 1     # the components did end differently


def check_max_iterations_next_to_early_stops(O, n_points=1200, max_iter=4):
    """One component runs into max_num_iterations while the others stop after at most two iterations: the done ones must not
    move again, and the loop keeps stepping the open one."""
    comps = [Comp(O, 2, [(1, 0)], cfg=21, start="solved", n_points=n_points),
             Comp(O, 4, synth.ring_edges(4, 2), cfg=22, n_points=n_points),
             Comp(O, 3, synth.ring_edges(3, 2), cfg=23, start="solved", n_points=n_points)]
    sums = check_batch(O, comps, PARAM_SE3, COST_P2PLANE, True, max_iter=max_iter)
    assert TERMINATION[sums[1]["termination"]] == "MAX_ITERATIONS" and sums[1]["num_iterations"] == max_iter, sums
    assert sums[0]["num_iterations"] <= 2 and sums[2]["num_iterations"] <= 2, sums


def test_max_iterations_next_to_early_stops(oracle):
    check_max_iterations_next_to_early_stops(oracle)


# ---- 3. storage modes ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", G.MODES)
@pytest.mark.parametrize("path", ["unit", "general"])
def test_storage_modes(oracle, mode, path):
    comps = mixed_comps(oracle, n_points=1000, nonrigid=path == "general", mode=mode, wide=False)
    for param, cost in ((PARAM_SE3, COST_P2P), (PARAM_QUAT, COST_P2PLANE if mode != "f32_no_normals" else COST_P2P)):
        check_batch(oracle, comps, param, cost, True, mode=mode)


# ---- 4. ICP rounds: correspond + optimize_components -----------------------------------------------------------------
def check_icp_rounds(n_pairs=8, n_points=3000, rounds=20, thresh=0.05):
    """`rounds` rounds of correspond + optimize_components on a batch of two-view problems equal a fresh engine per pair
    running correspond + optimize.  The second half of the rounds runs one LM iteration each, as a converged ICP loop does, so
    the correspondence step takes its cross-round shortcuts (certified matches, guessed median select)."""
    pairs = [scene(2, n_points, 100 + i) for i in range(n_pairs)]
    edges = [(1, 0), (0, 1)]
    M = 2 * n_pairs
    # pair i: frames i and n_pairs + i (interleaved); its edges (n_pairs + i -> i), (i -> n_pairs + i)
    pts = [p["pts"][0] for p in pairs] + [p["pts"][1] for p in pairs]
    nor = [p["nor"][0] for p in pairs] + [p["nor"][1] for p in pairs]
    poses = np.concatenate([np.stack([p["poses_init"][0] for p in pairs]), np.stack([p["poses_init"][1] for p in pairs])])
    g_edges = [(n_pairs + i, i) for i in range(n_pairs)] + [(i, n_pairs + i) for i in range(n_pairs)]
    fx = [1] * n_pairs + [0] * n_pairs
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(g_edges); eng.set_poses(poses, fx)
    fresh = []
    for p in pairs:
        f = Engine(); f.set_frames(p["pts"], p["nor"]); f.set_graph(edges); f.set_poses(p["poses_init"]); fresh.append(f)
    assert G.tile_len(n_points * n_pairs) == G.tile_len(n_points)
    one = default_options(); one.max_num_iterations = 1
    for rnd in range(rounds):
        o = one if rnd >= rounds // 2 else None
        eng.correspond(thresh)
        summ = eng.optimize_components(PARAM_SE3, COST_P2PLANE, True, options=o)
        P = eng.get_poses()
        for i, f in enumerate(fresh):
            f.correspond(thresh)
            s = f.optimize(PARAM_SE3, COST_P2PLANE, True, options=o)
            assert summ[i] == s, (rnd, i, summ[i], s)
            assert np.array_equal(_bits(P[[i, n_pairs + i]]), _bits(f.get_poses())), (rnd, i)
    st = eng.stats()
    assert st["cert_rounds"] > 0, st
    for f in [eng] + fresh:
        f.close()
    return st


def test_icp_rounds_equal_one_engine_per_pair():
    check_icp_rounds()


# ---- 5. API ----------------------------------------------------------------------------------------------------------------
def check_api(n_points=500):
    sc = scene(7, n_points, 31)
    eng = Engine()
    with pytest.raises(MvicpError) as ei:
        eng.components()
    assert ei.value.code == 4
    eng.set_frames(sc["pts"], None)
    n, comp = eng.components()            # no graph: every frame is a component of its own
    assert n == 7 and list(comp) == list(range(7))
    with pytest.raises(MvicpError) as ei:
        eng.optimize_components(PARAM_SE3, COST_P2P, True)     # no graph yet
    assert ei.value.code == 4
    edges = [(3, 1), (5, 3), (2, 6)]
    eng.set_graph(edges)
    n, comp = eng.components()
    assert n == 4 and list(comp) == [0, 1, 2, 1, 3, 1, 2]
    for args in ((3, COST_P2P), (PARAM_SE3, 3), (-1, COST_P2P)):
        with pytest.raises(MvicpError) as ei:
            eng.optimize_components(args[0], args[1], True)
        assert ei.value.code == 1
    with pytest.raises(MvicpError) as ei:
        eng.optimize_components(PARAM_SE3, COST_P2PLANE, True)  # point-to-plane without normals
    assert ei.value.code == 1
    # the lowest frame of every component becomes fixed: its out-edges are no longer searched (edge 2 -> 6 here)
    eng.set_poses(sc["poses_init"], [0] * 7)
    eng.correspond(0.05)
    assert eng.stats()["queries"] == 3 * n_points
    s = eng.optimize_components(PARAM_SE3, COST_P2P, True)
    assert len(s) == 4 and s[0] == NO_UNKNOWNS and s[3] == NO_UNKNOWNS
    eng.correspond(0.05)
    assert eng.stats()["queries"] == 2 * n_points
    P = eng.get_poses()
    for f in (0, 4):                      # components without unknowns pass their poses through
        assert np.array_equal(_bits(P[f]), _bits(sc["poses_init"][f])), f
    for f in (1, 2):                      # the lowest frames of solved ones only take the parameter round trip
        assert pose_rel_err(P[f:f + 1], sc["poses_init"][f:f + 1]) <= 1e-14, f
    eng.set_poses(P, [0] * 7)             # set_poses frees them again
    eng.correspond(0.05)
    assert eng.stats()["queries"] == 3 * n_points
    eng.set_poses(P, [1] * 7)             # everything fixed: nothing moves, every component reports no unknowns
    assert eng.optimize_components(PARAM_SE3, COST_P2P, True) == [NO_UNKNOWNS] * 4
    assert np.array_equal(_bits(eng.get_poses()), _bits(P))
    eng.close()


def test_api():
    check_api()
