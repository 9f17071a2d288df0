"""GPU parity of the g2o backend (mvicp_optimize_g2o / mvicp_pairwise_g2o; icp-g2o.cpp) against the numpy restatement in
tests/g2o_model.py, on identical correspondences.

Parity contract.  At convergence g2o's acceptance test (rho > 0) and the outer loop's (impr > 0) decide on chi2 differences at
the rounding level, so equal numbers of calls and trials after that point cannot be required.  Required instead:
  * the trial trace (lambda, chi, tchi, rho, accepted) equals the model's step for step for as long as |chi - tchi| > 1e-9 chi
    and chi > 1e-20 chi2_initial (below that an exact fit has been reached and chi2 is rounding noise): the same accept /
    reject decisions and lambda within 1e-9 relative;
  * the final chi2 within 1e-9 relative, the final poses within 1e-8;
  * two runs of the engine bit-identical (poses, chi2 per call and trace);
  * a build and a trial evaluation at the same poses give the same chi2 bits (the trace's chi after an accepted trial is its
    tchi, after a rejected one the same chi; chi2 at the start of every call is the chi of a trace row)."""
import numpy as np
import pytest

import g2o_model as G
from helpers import pose_rel_err, rot_err_deg, scene
from mv_lm_icp_b200 import COST_P2P, COST_P2PLANE, Engine, ICP_G2O, synth

pytestmark = pytest.mark.gpu
BUMP = np.array([[1, -0.004, 0.003], [0.004, 1, -0.002], [-0.003, 0.002, 1]])   # not a rotation: a non-rigid pose


def check_against_model(eng, pts, nor, poses, edges, fixed, cost, options=None):
    """Run the engine's g2o solve on the correspondences it holds and the model on the same ones; assert the contract.
    Returns the engine's poses."""
    corr = []
    for e in range(len(edges)):
        f, s, _, _ = eng.get_edge(e)
        corr.append((f, s))
    eng.set_poses(poses, fixed)
    summ, chis = eng.optimize_g2o(cost, options)
    P = eng.get_poses(); trace = eng.g2o_trace()
    fx = [bool(v) for v in fixed]; fx[0] = True
    prob = G.Problem(pts, nor, edges, corr, fx, cost == COST_P2PLANE, eps=0.01 if options is None else options.information_eps)
    kw = {} if options is None else dict(iterations=options.iterations_per_call, max_calls=options.max_calls,
                                         no_improvement_limit=options.no_improvement_limit, max_trials=options.max_trials,
                                         tau=options.tau, ortho_after=options.orthonormalize_after)
    Pm, sm, chim, trm = G.optimize(prob, poses, **kw)
    assert summ["chi2_initial"] == pytest.approx(sm["chi2_initial"], rel=1e-12)
    k = 0
    floor = 1e-20 * sm["chi2_initial"]   # an exact fit: chi2 itself is rounding noise below this
    decided = lambda t, i: abs(t[i, 1] - t[i, 2]) > 1e-9 * t[i, 1] and t[i, 1] > floor   # noqa: E731
    while k < min(len(trace), len(trm)) and decided(trm, k) and decided(trace, k):
        assert trace[k, 4] == trm[k, 4], (k, trace[k], trm[k])
        assert abs(trace[k, 0] - trm[k, 0]) <= 1e-9 * trm[k, 0], (k, trace[k], trm[k])
        k += 1
    assert k >= 1
    assert abs(summ["chi2_final"] - sm["chi2_final"]) <= 1e-9 * max(sm["chi2_final"], 1e-300) + 1e-24, (summ, sm)
    assert abs(chis[-1] - summ["chi2_final"]) == 0.0
    assert pose_rel_err(P, Pm) <= 1e-8
    for f in range(len(pts)):          # frames outside the problem keep their pose bit for bit
        if f not in prob.col:
            assert np.array_equal(P[f], np.asarray(poses[f])), f
    assert summ["trials"] == len(trace) and summ["calls"] == len(chis) - 1
    # a build and a trial evaluation at the same poses give the same chi2 bits (every rho compares the two): after an accepted
    # trial the next row's chi is that trial's tchi; after a rejected one it is the same chi (the same iteration, or a rebuild
    # at the same estimate); and chi2 at the start of every call is the chi of a row, the first of that call
    for r in range(len(trace) - 1):
        assert trace[r + 1, 1] == (trace[r, 2] if trace[r, 4] else trace[r, 1]), (r, trace[r], trace[r + 1])
    r = 0
    for c in range(len(chis) - 1):
        while r < len(trace) and trace[r, 1] != chis[c]:
            r += 1
        assert r < len(trace), (c, chis[c])
    # a second run from the same start is bit-identical
    eng.set_poses(poses, fixed)
    summ2, chis2 = eng.optimize_g2o(cost, options)
    assert np.array_equal(eng.get_poses(), P) and np.array_equal(chis2, chis) and np.array_equal(eng.g2o_trace(), trace)
    assert summ2 == summ
    return P, summ, trace


def synthetic(n_views, n_points, cfg, fp64, nonrigid):
    sc = scene(n_views, n_points, cfg)
    pts = [p.copy() for p in sc["pts"]]; nor = [n.copy() for n in sc["nor"]]
    if fp64:   # coordinates no longer fp32-representable: the fp64 record storage
        pts = [p + 1e-9 * np.sin(np.arange(p.size)).reshape(p.shape) for p in pts]
    poses = sc["poses_init"].copy()
    if nonrigid:
        for f in range(1, n_views):
            poses[f][:3, :3] = poses[f][:3, :3] @ BUMP
    return pts, nor, poses


@pytest.mark.parametrize("cost", [COST_P2P, COST_P2PLANE])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("nonrigid", [False, True])
def test_ring_matches_model(cost, fp64, nonrigid, n_views=4, n_points=1500):
    pts, nor, poses = synthetic(n_views, n_points, 31, fp64, nonrigid)
    edges = synth.ring_edges(n_views, 2)
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges); eng.set_poses(poses)
    eng.correspond(0.05)
    fixed = np.zeros(n_views, np.uint8); fixed[0] = 1
    check_against_model(eng, pts, nor, poses, edges, fixed, cost)
    eng.close()


@pytest.mark.parametrize("cost", [COST_P2P, COST_P2PLANE])
def test_loop_closure_second_fixed_frame_and_an_empty_frame(cost, n_points=1500):
    """Ring of 6 with a loop-closure chord 5 -> 1, frames 0 and 3 fixed (edges into and out of frame 3 included, an edge
    between the two fixed frames is not active), and frame 4 free without a single correspondence: it is not a vertex of the
    problem and keeps its pose bit for bit."""
    n_views = 6
    pts, nor, poses = synthetic(n_views, n_points, 33, False, False)
    edges = synth.ring_edges(n_views, 2) + [(5, 1), (3, 0)]
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges)
    fixed = np.zeros(n_views, np.uint8); fixed[0] = 1
    eng.set_poses(poses, fixed)
    eng.correspond(0.05)
    for e, (s, d) in enumerate(edges):
        if s == 3 and d == 0:
            eng.set_edge(e, np.arange(50), np.arange(50), 0.0)   # between two fixed frames once frame 3 is fixed
        if 4 in (s, d):
            eng.set_edge(e, [], [], 0.0)
    fixed[3] = 1
    P, _, _ = check_against_model(eng, pts, nor, poses, edges, fixed, cost)
    assert np.array_equal(P[4], poses[4]) and np.array_equal(P[3], poses[3]) and np.array_equal(P[0], poses[0])
    eng.close()


@pytest.mark.parametrize("cost", [COST_P2P, COST_P2PLANE])
def test_real_bunny_nonrigid_poses(golden_dir, cost):
    """The reference's own scans under their non-rigid Bunny_RealData sample poses (fp64 storage): the isometry inverse uses
    the transpose of the non-orthogonal 3x3 part and J_dst keeps g2o's -I, exactly as the model does."""
    g = np.load(f"{golden_dir}/bunny_pair.npz")
    pts = [g["pts0"], g["pts1"], g["pts0"][::2].copy()]; nor = [g["nor0"], g["nor1"], g["nor0"][::2].copy()]
    bump = np.eye(4); bump[:3, :3] = BUMP; bump[:3, 3] = [0.002, -0.001, 0.0015]
    poses = np.stack([g["pose0"], g["pose1"], bump @ g["pose0"]])
    edges = [(1, 0), (1, 2), (2, 1), (2, 0)]
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges); eng.set_poses(poses)
    eng.correspond(0.05)
    check_against_model(eng, pts, nor, poses, edges, np.array([1, 0, 0], np.uint8), cost)
    eng.close()


def _noisy_pairwise(golden_dir):
    """main_pairwise.cpp:34-60 on cloudXYZ_0: P = addNoise(Translation(tra) * q, 0.1, 0.1); the noisy P is stored here."""
    g = np.load(f"{golden_dir}/bunny_pair.npz")
    src, nor = g["pts0"], g["nor0"]
    P = np.array([[0.52369438, 0.18219566, 0.83219287, 0.06273934],
                  [0.57958032, 0.65155938, -0.48953148, -0.08017062],
                  [-0.62142578, 0.73637498, 0.26504412, 0.03651208],
                  [0.0, 0.0, 0.0, 1.0]])
    U, _, Vt = np.linalg.svd(P[:3, :3]); P[:3, :3] = U @ Vt   # an exact rotation
    return src, nor, P


@pytest.mark.parametrize("cost", [COST_P2P, COST_P2PLANE])
def test_pairwise_known_answer(golden_dir, cost):
    """ICP_G2O::pointToPoint / pointToPlane recover P (README.md:150 reports 6.4e-17 m / 0 degrees for g2o)."""
    src, nor, P = _noisy_pairwise(golden_dir)
    dst = src @ P[:3, :3].T + P[:3, 3]; ndst = nor @ P[:3, :3].T
    Pe, s = ICP_G2O.pointToPlane(src, dst, ndst) if cost == COST_P2PLANE else ICP_G2O.pointToPoint(src, dst)
    # rotation angle from |R - I|_F / sqrt(2): arccos of the trace (rot_err_deg) cannot resolve angles below ~1e-6 degrees
    ang = np.degrees(np.linalg.norm(Pe[:3, :3] @ P[:3, :3].T - np.eye(3)) / np.sqrt(2))
    assert np.linalg.norm(Pe[:3, 3] - P[:3, 3]) <= 1e-10 and ang <= 1e-6 and rot_err_deg(Pe, P) < 1e-5, (Pe, P, ang)
    assert s["calls"] == 1 and s["iterations"] <= 300 and s["accepted"] >= 1
    prob = G.Problem([dst, src], [ndst, ndst], [(1, 0)], [(np.arange(len(src)), np.arange(len(src)))], [True, False],
                     cost == COST_P2PLANE)
    Pm, sm, _, _ = G.optimize(prob, [np.eye(4), np.eye(4)], iterations=300, max_calls=1)
    assert np.max(np.abs(Pe - Pm[1])) <= 1e-8


def test_options_and_errors():
    pts, nor, poses = synthetic(3, 800, 35, False, False)
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(synth.ring_edges(3, 2)); eng.set_poses(poses)
    eng.correspond(0.05)
    from mv_lm_icp_b200 import COST_MIXED, MvicpError, default_g2o_options
    with pytest.raises(MvicpError) as ei:
        eng.optimize_g2o(COST_MIXED)
    assert ei.value.code == 1
    o = default_g2o_options()
    assert (o.iterations_per_call, o.max_calls, o.no_improvement_limit, o.max_trials, o.orthonormalize_after) == (100, 100, 5, 10, 1000)
    assert (o.tau, o.information_eps) == (1e-5, 0.01)
    o.max_calls = 2; o.iterations_per_call = 3
    fixed = np.array([1, 0, 0], np.uint8)
    _, s, _ = check_against_model(eng, pts, nor, poses, synth.ring_edges(3, 2), fixed, COST_P2PLANE, o)
    assert s["calls"] <= 2 and s["iterations"] <= 6
    eng.close()


@pytest.mark.parametrize("ortho_after", [1000, 2])
def test_rejected_trials_and_orthonormalisation(ortho_after):
    """The problem of the committed trace (tests/golden/g2o_trace.npz): a strongly non-rigid free dst frame makes trials overshoot,
    so rejections (lambda *= nu, nu *= 2, the undo) run on the device.  With orthonormalize_after = 2 the counter -- which also
    counts rejected trials -- fires every third update of a vertex and the re-orthonormalised poses are compared with the
    model's."""
    from mv_lm_icp_b200 import default_g2o_options
    from test_g2o_model import golden_problem
    pts, nor, edges, corr, start = golden_problem()
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges)
    for e, (f, s) in enumerate(corr):
        eng.set_edge(e, f, s, 1.0)
    o = default_g2o_options(); o.orthonormalize_after = ortho_after
    _, s, trace = check_against_model(eng, pts, nor, np.stack(start), edges, np.array([1, 0, 0], np.uint8), COST_P2PLANE, o)
    assert (trace[:, 4] == 0).sum() >= 5 and s["accepted"] >= 5
    eng.close()


@pytest.mark.parametrize("scale", [1.3, 0.7])
def test_non_unit_normals(scale, n_views=4, n_points=1500):
    """prec0 from normals that are not unit: R0^T diag(eps, eps, 1) R0 differs from eps I + (1 - eps) n n^T there, and the
    engine must build the former (the model does; tests/test_g2o_model.py checks that the two differ)."""
    pts, nor, poses = synthetic(n_views, n_points, 37, False, False)
    nor = [n * scale for n in nor]
    edges = synth.ring_edges(n_views, 2)
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges); eng.set_poses(poses)
    eng.correspond(0.05)
    fixed = np.zeros(n_views, np.uint8); fixed[0] = 1
    check_against_model(eng, pts, nor, poses, edges, fixed, COST_P2PLANE)
    eng.close()
