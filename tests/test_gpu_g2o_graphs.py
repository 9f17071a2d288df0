"""GPU parity of the g2o solve (mvicp_optimize_g2o) on every storage mode, on arbitrary pose graphs and fixed-frame sets, at the
streaming tile boundaries, and on the branches a converging solve does not take (a failed factorisation, |q|^2 > 1, degenerate
makeRot0 normals) -- against tests/g2o_model.py on identical correspondences, under the contract of tests/test_gpu_g2o.py
(check_against_model: trial trace while decided, lambda and final chi2 within 1e-9, poses within 1e-8, frames outside the
problem bit for bit, two runs bit-identical, build and trial chi2 the same bits).  chi2 at the start point is a direct readout
of g2o_eval_kernel + g2o_edge_kernel and is held to 1e-12 relative, against the model and against a math.fsum of
per-correspondence terms with makeRot0 / prec0 written out."""
import math

import numpy as np
import pytest

import g2o_model as G
from helpers import oracle_correspond, scene
from mv_lm_icp_b200 import COST_P2P, COST_P2PLANE, PARAM_SE3, Engine, MvicpError, default_g2o_options, synth
from test_gpu_g2o import check_against_model, synthetic
from test_gpu_lm_graphs import (FIXED_SETS, HUB_RING, MODES, OFF_GRID, SMEM_LIMIT, TOPOLOGIES, _f32_exact, _nonrigid, _rigid,
                                _storage_setup, tile_len, tile_scene, topology, wide_graph)

pytestmark = pytest.mark.gpu
READOUT_TOL = 1e-12
ERR_INVALID = 1                                  # include/mvicp.h: MVICP_ERR_INVALID
END_NO_IMPROVEMENT, END_NO_VERTICES = 0, 2       # MVICP_G2O_END_*
CALL_TERMINATE = 0                               # MVICP_G2O_CALL_TERMINATE
EMPTY = (np.zeros(0, np.int32), np.zeros(0, np.int32))


def short_options(max_calls=1, iterations=8):
    """Bounded solves for the graph cases.  Near the optimum chi2 resolves a pose only to ~sqrt(1e-16 chi2 / H), and g2o
    keeps accepting steps whose rho is rounding noise: past the decided trials engine and model would wander apart by more
    than the 1e-8 pose bar (chi2 itself stays within 1e-9).  These cases stop while the trials are still decided."""
    o = default_g2o_options(); o.max_calls = max_calls; o.iterations_per_call = iterations
    return o


# ---- helpers ---------------------------------------------------------------------------------------------------------
def fixed_flags(M, fixed):
    fx = np.zeros(M, np.uint8)
    fx[list(fixed)] = 1
    fx[0] = 1                       # g2oOptimizer fixes frame 0 itself (icp-g2o.cpp:182-186)
    return fx


def upload(eng, corr):
    for e, (f, s) in enumerate(corr):
        eng.set_edge(e, f, s, 1.0)


def readout_options():
    """One call of one iteration of one trial: the solve's chi2_initial is the first build evaluation."""
    o = default_g2o_options()
    o.max_calls = o.iterations_per_call = o.max_trials = 1
    return o


def g2o_profile(M, edges, counts, fixed):
    """g2o's columns and row profile (mvicp_optimize_g2o): an edge is active when it has a correspondence and a free end, a
    frame has a column when it is free and an end of an active edge (columns in frame order), and every row of a block starts
    at the lowest column of a frame it shares an active edge with.  Returns (col, rfirst, n, active edges)."""
    fx = fixed_flags(M, fixed)
    act = [e for e, (s, d) in enumerate(edges) if counts[e] and not (fx[s] and fx[d])]
    touched = {v for e in act for v in edges[e]}
    col, n = {}, 0
    for f in range(M):
        if f in touched and not fx[f]:
            col[f] = n; n += 6
    rfirst = [(r // 6) * 6 for r in range(n)]
    for e in act:
        s, d = edges[e]
        if s in col and d in col:
            lo, hi = sorted((col[s], col[d]))
            for i in range(6):
                rfirst[hi + i] = min(rfirst[hi + i], lo)
    return col, rfirst, n, act


def skyline_bytes(rfirst, n):
    """Bytes g2o_step_kernel needs for the skyline factor and its vectors (run_steps: shared memory up to SMEM_LIMIT)."""
    return 8 * (sum(r - rfirst[r] + 1 for r in range(n)) + n) + 8 * 3 * (n + 1)


def chi2_fsum(pts, nor, poses, edges, corr, fixed, plane, eps=0.01):
    """chi2 = sum e^T R0^T diag(eps, eps, 1) R0 e = sum_k d_k (R0_k . e)^2 per correspondence, summed with math.fsum; R0 from
    makeRot0 written out: row 2 = n, row 1 = normalise((0,1,0) - n_y n) (a zero vector stays zero), row 0 = n x row 1."""
    terms = []
    for (s, d), (f, sec) in zip(edges, corr):
        if not len(f) or (fixed[s] and fixed[d]):
            continue
        F0, t0, F1, t1 = poses[d][:3, :3], poses[d][:3, 3], poses[s][:3, :3], poses[s][:3, 3]
        e = (pts[s][f] @ F1.T + t1 - t0) @ F0 - pts[d][sec]
        if plane:
            n = nor[d][sec]
            y = np.stack([-n[:, 1] * n[:, 0], 1.0 - n[:, 1] * n[:, 1], -n[:, 1] * n[:, 2]], axis=1)
            ny = np.sqrt(np.sum(y * y, axis=1))
            y = y / np.where(ny > 0, ny, 1.0)[:, None]
            x = np.cross(n, y)
            q = eps * np.sum(x * e, axis=1) ** 2 + eps * np.sum(y * e, axis=1) ** 2 + np.sum(n * e, axis=1) ** 2
        else:
            q = np.sum(e * e, axis=1)
        terms.extend(q.tolist())
    return math.fsum(terms)


def check_readout(eng, pts, nor, poses, edges, corr, fx, cost, what):
    """chi2 at the start point against the model and the fsum evaluation; chi2 before the first call is that number."""
    eng.set_poses(poses, fx)
    s, chis = eng.optimize_g2o(cost, readout_options())
    plane = cost == COST_P2PLANE
    want = G.Problem(pts, nor, edges, corr, [bool(v) for v in fx], plane).chi2(list(poses))
    c_np = chi2_fsum(pts, nor, poses, edges, corr, fx, plane)
    assert chis[0] == s["chi2_initial"] and s["calls"] == 1 and s["trials"] == 1, (what, s)
    assert abs(s["chi2_initial"] - want) <= READOUT_TOL * want, (what, s["chi2_initial"], want)
    assert abs(s["chi2_initial"] - c_np) <= READOUT_TOL * c_np, (what, s["chi2_initial"], c_np)


# ---- 1. storage modes x cost x rigid / non-rigid poses -----------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("path", ["unit", "general"])
def test_storage_modes_match_model(oracle, mode, path):
    """fp32 records with packed normals, fp32 points with recomputed fp64 normals (g2o_eval_kernel<true, false, P2PLANE>),
    fp64 records, and fp32 without normals, where point-to-plane is refused; rigid ("unit") and non-rigid ("general") poses.
    _storage_setup asserts the input property that selects each mode."""
    eng, pts, nor, poses, edges, corr, _ = _storage_setup(oracle, mode, path)
    upload(eng, corr)
    fx = fixed_flags(len(pts), (0,))
    check_against_model(eng, pts, nor, poses, edges, fx, COST_P2P)
    if mode == "f32_no_normals":
        with pytest.raises(MvicpError) as ei:
            eng.optimize_g2o(COST_P2PLANE)
        assert ei.value.code == ERR_INVALID
    else:
        check_against_model(eng, pts, nor, poses, edges, fx, COST_P2PLANE)
    eng.close()


# ---- 2. graph topologies ---------------------------------------------------------------------------------------------
def g2o_topology(name):
    """(n_views, edges, fixed frames, frames whose edges carry no inlier, whether edges out of frame 0 carry matches)."""
    if name == "mid_empty":           # frame 5, free and mid-order, has edges without inliers: no column, later columns shift
        M, edges, fixed = topology("ring_chord")
        return M, edges, fixed, {5}, False
    if name == "fixed_src":           # edges out of the fixed frames 0 and 4 carry matches: active in g2o, dropped by LM
        M, edges, _ = topology("ring_chord")
        return M, edges, (0, 4), set(), True
    M, edges, fixed = topology(name)
    return M, edges, fixed, set(), False


G2O_TOPOLOGIES = TOPOLOGIES + ["mid_empty", "fixed_src"]


def graph_corr(O, pts, poses, edges, empty=(), src0=False):
    """The oracle's correspondence step on every edge (edges out of frame 0 only with src0); edges touching `empty` get none."""
    ref = oracle_correspond(O, pts, poses, edges, fixed0=not src0)
    corr = [((r["first"], r["second"]) if r else EMPTY) for r in ref]
    return [EMPTY if (s in empty or d in empty) else c for (s, d), c in zip(edges, corr)]


def run_graph(O, M, edges, fixed, empty=(), src0=False, n_points=1500, cfg=43, rounds=2, cost=COST_P2PLANE, views=None,
              options=None, check=None):
    """Consecutive g2o solves on one engine, each from the previous solve's poses with fresh oracle correspondences; frame f is
    the scene's view views[f] (default: view f).  check(corr) asserts the structure of the first round."""
    sc = scene(M, n_points, cfg)
    order = list(range(M)) if views is None else [views.index(f) for f in range(M)]
    pts, nor = [sc["pts"][v] for v in order], [sc["nor"][v] for v in order]
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges)
    poses = sc["poses_init"][order].copy()
    fx = fixed_flags(M, fixed)
    for rnd in range(rounds):
        corr = graph_corr(O, pts, poses, edges, empty, src0)
        if check is not None and rnd == 0:
            check(corr)
        upload(eng, corr)
        poses, _, _ = check_against_model(eng, pts, nor, poses, edges, fx, cost, short_options() if options is None else options)
    eng.close()


@pytest.mark.parametrize("name", G2O_TOPOLOGIES)
def test_graph_topologies_match_model(oracle, name):
    M, edges, fixed, empty, src0 = g2o_topology(name)
    fx = fixed_flags(M, fixed)

    def check(corr):
        col, rfirst, n, act = g2o_profile(M, edges, [len(f) for f, _ in corr], fixed)
        starts = [rfirst[r] // 6 for r in range(0, n, 6)]     # first block column of every block row
        if name == "hub_last":        # one wide block row at the end; rows before it that do not reach the previous block
            assert starts[-1] == 0 and any(starts[b] == b for b in range(1, len(starts) - 1)), starts
        if name == "ring_chord":      # the chord's row reaches four blocks back
            assert starts[5] == 1, starts
        if name.startswith("random"):
            assert edges != sorted(edges)
        if name == "two_components":  # no row of the second ring reaches into the first
            assert all(starts[col[f] // 6] >= col[6] // 6 for f in range(6, 10)), starts
        if name == "dst_only":        # frames that are never a src still get a column
            assert 3 in col and 6 in col and not any(edges[e][0] in (3, 6) for e in act)
        if name == "dst_fixed":       # the fixed frame 4 has no column; its out-edges are active
            assert 4 not in col and any(edges[e][0] == 4 for e in act)
        if name == "mid_empty":       # frame 5 has no column: frame 6 takes the one LM gives frame 5
            assert 5 not in col and col[6] == 24 and n == 6 * (M - 2)
        if name == "fixed_src":       # active edges out of both fixed frames
            assert {edges[e][0] for e in act if fx[edges[e][0]]} == {0, 4}
    run_graph(oracle, M, edges, fixed, empty=empty, src0=src0, views=HUB_RING if name == "hub_last" else None, check=check)


# ---- 3. the factor in global memory ------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_views,over", [(36, False), (48, True)])
def test_wide_graph_factor_in_global_memory(oracle, n_views, over):
    """g2o_step_kernel keeps the skyline factor in global memory when it and its vectors exceed 220 KiB: the wide graph's
    profile over g2o's own column set needs ~320 KiB at 48 views and ~180 KiB at 36."""
    edges = wide_graph(n_views)
    o = short_options()

    def check(corr):
        col, rfirst, n, _ = g2o_profile(n_views, edges, [len(f) for f, _ in corr], (0,))
        assert n == 6 * (n_views - 1)
        assert (skyline_bytes(rfirst, n) > SMEM_LIMIT) == over, skyline_bytes(rfirst, n)
    run_graph(oracle, n_views, edges, (0,), rounds=1, options=o, check=check)


# ---- 4. fixed-frame sets ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fixed", FIXED_SETS, ids=lambda f: "fixed" + "_".join(map(str, f)))
def test_fixed_sets_match_model(oracle, fixed):
    M, edges, _ = topology("ring_chord")
    run_graph(oracle, M, edges, fixed, rounds=1, cost=COST_P2P)


def test_all_frames_fixed_leaves_poses_unchanged(oracle):
    M, edges, _ = topology("ring_chord")
    sc = scene(M, 1500, 43)
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges)
    upload(eng, graph_corr(oracle, sc["pts"], sc["poses_init"], edges))
    eng.set_poses(sc["poses_init"], [1] * M)
    s, chis = eng.optimize_g2o(COST_P2PLANE)
    assert s["ended"] == END_NO_VERTICES and s["calls"] == 0 and s["trials"] == 0 and chis.tolist() == [0.0], (s, chis)
    assert len(eng.g2o_trace()) == 0
    assert np.array_equal(eng.get_poses().view(np.uint64), np.asarray(sc["poses_init"]).view(np.uint64))
    eng.close()


def test_switching_fixed_sets_between_solves(oracle):
    """One engine, the fixed set changed before every solve: each change lays the work out again.  Second part: tile_scene(2048),
    where fixing the 1.1 M-point frame 5 drops the tile length to 1024 and its edge into the free frame 1 stays active."""
    M, edges, _ = topology("ring_chord")
    sc = scene(M, 1500, 43)
    poses = sc["poses_init"]
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges)
    upload(eng, graph_corr(oracle, sc["pts"], poses, edges))
    for fixed in [(0,), (0, 4), (0, 2, 5), (0,), (0, 7), (0, 4)]:
        check_against_model(eng, sc["pts"], sc["nor"], poses, edges, fixed_flags(M, fixed), COST_P2PLANE, short_options())
    eng.close()
    pts, nor, poses, edges, corr, _, _ = tile_scene(2048)
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges)
    upload(eng, corr)
    o = short_options(1, 5)
    seen = []
    for fixed in [(0,), (0, 5), (0, 2), (0, 2, 5), (0,)]:
        fx = fixed_flags(len(pts), fixed)
        seen.append(tile_len(sum(len(pts[s]) for s, _ in edges if not fx[s])))
        check_against_model(eng, pts, nor, poses, edges, fx, COST_P2PLANE, o)
    assert seen == [2048, 1024, 2048, 1024, 2048], seen
    eng.close()


# ---- 5. tile boundaries and the chi2 readout ---------------------------------------------------------------------------
def g2o_tile_scene(tl):
    """tile_scene(tl) plus two edges out of the fixed frame 0 (3001 points) with inliers on the first and last slot of each of
    its tiles: active in the g2o solve, not counted by the tile length, which counts the slots of free src frames only."""
    pts, nor, poses, edges, corr, _, active = tile_scene(tl)
    assert tile_len(active) == tl, (active, tile_len(active))
    n0 = len(pts[0])
    ends = np.array(sorted({k for t in range(0, n0, tl) for k in (t, min(t + tl, n0) - 1)}), np.int32)
    rng = np.random.default_rng(tl)
    extra = [(0, 1), (0, 4)]
    corr = corr + [(ends, rng.integers(0, len(pts[d]), len(ends)).astype(np.int32)) for _, d in extra]
    edges = edges + extra
    assert sum(len(pts[s]) for s, _ in edges if s != 0) == active and tile_len(active + len(extra) * n0) == tl
    return pts, nor, poses, edges, corr


def check_tile_readout(O, tl, modes=MODES, nonrigid=(False, True)):
    pts0, nor0, poses0, edges, corr = g2o_tile_scene(tl)
    fx = fixed_flags(len(pts0), (0,))
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
        upload(eng, corr)
        costs = [COST_P2P] if mode == "f32_no_normals" else [COST_P2P, COST_P2PLANE]
        for nr in nonrigid:
            poses = poses0.copy()
            if nr:
                poses[1] = _nonrigid(poses[1])
            for cost in costs:
                check_readout(eng, pts, nor, poses, edges, corr, fx, cost, (tl, mode, nr, cost))
        # one full iteration: the normal matrix and gradient behind the first step
        o = default_g2o_options(); o.max_calls = 1; o.iterations_per_call = 1
        check_against_model(eng, pts, nor, poses0, edges, fx, costs[-1], o)
        eng.close()


@pytest.mark.parametrize("tl", [1024, 2048, 4096, 8192])
def test_tile_boundaries_chi2_readout(oracle, tl):
    check_tile_readout(oracle, tl)


# ---- 6. (build and trial chi2: check_against_model) -- 7. a failed factorisation ---------------------------------------
def _two_frames(rng, n=300):
    dst = (rng.normal(size=(n, 3)) * 0.1).astype(np.float32).astype(np.float64)
    src = (rng.normal(size=(n, 3)) * 0.1).astype(np.float32).astype(np.float64)
    return dst, src


@pytest.mark.parametrize("ortho_after", [1000, 2])
def test_failed_factorisation_is_a_rejected_trial(ortho_after):
    """Every match's src point sits exactly at the origin, so J_src's rotation columns and H's rotation block are exactly zero;
    with tau = 0 (lambda = 0) the fourth pivot is exactly zero.  Every trial is then rejected without an evaluation (tchi =
    +inf, rho = -inf), lambda stays 0, each call ends on Terminate, the outer loop on no improvement, and the pose is kept."""
    rng = np.random.default_rng(17)
    dst, src = _two_frames(rng)
    src[:40] = 0.0
    pts, nor = [dst, src], [None, None]
    poses = np.stack([np.eye(4), _rigid(rng, 0.05, 0.02)])
    edges = [(1, 0)]
    corr = [(np.arange(40, dtype=np.int32), rng.choice(len(dst), 40, replace=False).astype(np.int32))]
    eng = Engine(); eng.set_frames(pts, None); eng.set_graph(edges); upload(eng, corr)
    o = default_g2o_options(); o.tau = 0.0; o.orthonormalize_after = ortho_after
    fx = np.array([1, 0], np.uint8)
    P, s, trace = check_against_model(eng, pts, nor, poses, edges, fx, COST_P2P, o)
    assert len(trace) and np.all(trace[:, 0] == 0.0) and np.all(trace[:, 2] == np.inf), trace
    assert np.all(trace[:, 3] == -np.inf) and np.all(trace[:, 4] == 0.0), trace
    assert s["ended"] == END_NO_IMPROVEMENT and s["last_call_end"] == CALL_TERMINATE and s["accepted"] == 0, s
    assert np.array_equal(P.view(np.uint64), poses.view(np.uint64))
    _, sm, _, trm = G.optimize(G.Problem(pts, nor, edges, corr, [True, False], False), poses, tau=0.0, ortho_after=ortho_after)
    model_evals = sm["iterations"] + int(np.sum(np.isfinite(trm[:, 2])))   # one build per iteration, one per evaluated trial
    assert (s["calls"], s["iterations"], s["trials"], s["evaluations"]) == (sm["calls"], sm["iterations"], sm["trials"], model_evals)
    assert s["trials"] == sm["calls"] * o.max_trials
    eng.close()


# ---- 8. |q|^2 > 1 ----------------------------------------------------------------------------------------------------
def test_rotation_increment_outside_the_unit_ball(monkeypatch):
    """dst is a x4 scaled, 90-degree rotated copy of src: the first Gauss-Newton rotation increments have |q|^2 ~ 4, where
    fromVectorMQT keeps the identity rotation.  The model is wrapped to confirm the branch runs on decided trials."""
    rng = np.random.default_rng(3)
    _, src = _two_frames(rng, 200)
    src = (src + 0.05).astype(np.float32).astype(np.float64)
    Rz = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    dst = 4.0 * src @ Rz.T
    assert _f32_exact(dst)
    pts, nor, edges = [dst, src], [None, None], [(1, 0)]
    idx = np.arange(len(src), dtype=np.int32)
    poses = np.stack([np.eye(4), np.eye(4)])
    o = default_g2o_options(); o.tau = 1e-3; o.max_calls = 1; o.iterations_per_call = 30   # every trial decided
    hits, real = [], G.increment

    def increment(d):
        hits.append(1.0 - (d[3] * d[3] + d[4] * d[4] + d[5] * d[5]) < 0)
        return real(d)
    monkeypatch.setattr(G, "increment", increment)
    _, _, _, trm = G.optimize(G.Problem(pts, nor, edges, [(idx, idx)], [True, False], False), poses, tau=o.tau, max_calls=1,
                              iterations=o.iterations_per_call)
    decided = np.abs(trm[:, 1] - trm[:, 2]) > 1e-9 * trm[:, 1]
    lead = int(np.argmin(decided)) if not decided.all() else len(decided)   # rows before the first undecided one
    assert len(hits) == len(trm) and sum(hits[:lead]) >= 5, (sum(hits), lead)
    monkeypatch.setattr(G, "increment", real)
    eng = Engine(); eng.set_frames(pts, None); eng.set_graph(edges); upload(eng, [(idx, idx)])
    check_against_model(eng, pts, nor, poses, edges, np.array([1, 0], np.uint8), COST_P2P, o)
    eng.close()


# ---- 9. makeRot0 edges ------------------------------------------------------------------------------------------------
def special_normals(nor, near_ey):
    """dst normals exactly zero, exactly (0, +-1, 0) -- makeRot0's zero row 1 -- and, with near_ey, (d, 1 - k 2^-53, d')
    where 1 - n_y^2 cancels."""
    out = []
    for f, n in enumerate(nor):
        n = n.copy()
        n[0::7] = 0.0
        n[1::11] = [0.0, 1.0, 0.0]
        n[2::13] = [0.0, -1.0, 0.0]
        if near_ey:
            m = len(n[3::5])
            k = 1 + np.arange(m) % 4
            n[3::5] = np.stack([np.array([0.0, 2.0 ** -60, 1e-9, -3e-17])[np.arange(m) % 4], 1.0 - k * 2.0 ** -53,
                                np.array([0.0, -2.0 ** -58, 2e-9, 0.0])[(np.arange(m) + f) % 4]], axis=1)
        out.append(n)
    return out


@pytest.mark.parametrize("near_ey", [False, True])
def test_makerot0_degenerate_normals(near_ey, n_views=4, n_points=1500):
    pts, nor, poses = synthetic(n_views, n_points, 31, False, False)
    nor = special_normals(nor, near_ey)
    assert all(_f32_exact(n) for n in nor) == (not near_ey)      # near e_y the normals (and so the records) are fp64
    edges = synth.ring_edges(n_views, 2)
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges); eng.set_poses(poses)
    eng.correspond(0.05)
    corr = [eng.get_edge(e)[:2] for e in range(len(edges))]
    used = np.concatenate([nor[d][sec] for (_, d), (_, sec) in zip(edges, corr)])
    assert (used == 0).all(axis=1).any() and (used == [0, 1, 0]).all(axis=1).any() and (used == [0, -1, 0]).all(axis=1).any()
    if near_ey:
        assert ((used[:, 1] < 1) & (used[:, 1] >= 1 - 4 * 2.0 ** -53)).sum() >= 100
    fx = fixed_flags(n_views, (0,))
    check_readout(eng, pts, nor, poses, edges, corr, fx, COST_P2PLANE, near_ey)
    check_against_model(eng, pts, nor, poses, edges, fx, COST_P2PLANE)
    eng.close()


# ---- 10. LM and g2o interleaved on one engine --------------------------------------------------------------------------
@pytest.mark.parametrize("recomputed", [False, True], ids=["packed_normals", "recomputed_normals"])
def test_lm_and_g2o_interleaved_on_one_engine(oracle, recomputed):
    """LM, g2o, LM, g2o on one engine (same correspondences, poses reset before each solve) equal, bit for bit, a fresh engine
    running each solve alone.  Frame 3 is free without correspondences: LM keeps its column, g2o drops it, so the two column
    sets differ while the fixed set -- and so LM's cached layout key -- stays the same."""
    M = 5
    sc = scene(M, 1500, 43)
    pts, poses = sc["pts"], sc["poses_init"]
    edges = synth.ring_edges(M, 2)
    ref = oracle_correspond(oracle, pts, poses, edges)
    corr = [EMPTY if (r is None or 3 in edges[e]) else (r["first"], r["second"]) for e, r in enumerate(ref)]
    w = [np.float32(0) if not len(c[0]) else np.float32(ref[e]["weight"]) for e, c in enumerate(corr)]
    fx = fixed_flags(M, (0,))
    col, _, n, _ = g2o_profile(M, edges, [len(f) for f, _ in corr], (0,))
    assert 3 not in col and n == 6 * (M - 2)                      # LM: 6 (M - 1) columns

    def fresh():
        eng = Engine(); eng.set_frames(pts, sc["nor"])
        if recomputed:
            nor, _ = eng.recompute_normals(10)
            assert not all(_f32_exact(v) for v in nor)
        eng.set_graph(edges)
        for e, (f, s) in enumerate(corr):
            eng.set_edge(e, f, s, w[e])
        return eng

    def solve(eng, kind):
        eng.set_poses(poses, fx)
        if kind == "lm":
            s = eng.optimize(PARAM_SE3, COST_P2PLANE, True)
            return eng.get_poses(), s
        s, chis = eng.optimize_g2o(COST_P2PLANE)
        return eng.get_poses(), s, chis, eng.g2o_trace()

    kinds = ["lm", "g2o", "lm", "g2o"]
    eng = fresh()
    got = [solve(eng, k) for k in kinds]
    eng.close()
    for k, g in zip(kinds, got):
        e2 = fresh(); want = solve(e2, k); e2.close()
        assert np.array_equal(g[0].view(np.uint64), want[0].view(np.uint64)), k
        assert g[1] == want[1], (k, g[1], want[1])
        if k == "g2o":
            assert np.array_equal(g[2], want[2]) and np.array_equal(g[3], want[3]), k
    assert not np.array_equal(got[0][0], got[1][0])               # the two solvers did move the poses differently
