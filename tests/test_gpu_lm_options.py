"""The LM trust-region loop (csrc/lm_step.cuh, lm_step_body) under non-default options and failing steps, on the joint path
(Engine.optimize) and the per-component path (Engine.optimize_components), against the oracle's Ceres-style loop
(oracle/lm.h, lm_minimize) run with the same option values; and the option rules of include/mvicp.h.

Bar, for every case: the bar of tests/test_gpu_lm_graphs.py (equal termination, iteration and successful-step counts, costs
within COST_TOL, poses within TIGHT_TOL -- here per frame, so that a frame placed far away does not hide the others) plus
the two counters the oracle does not report under the same names:
  num_evaluations   == 1 + the oracle's candidate evaluations: one streaming pass at the start point and one per candidate
                       the step kernel proposed (a failed factor or a non-positive model change proposes none);
  num_linear_solves == the oracle's iterations: one factorisation per step attempt.
Decision-margin guard, for every case: before the engine is compared, the oracle's loop is re-run with every threshold it
compares against (min_relative_decrease, function_tolerance, parameter_tolerance, gradient_tolerance,
min_trust_region_radius) moved by a relative 1e-6 either way; each run must take the same decisions (the trace's valid /
accepted columns, termination, counts).  A decision that a 1e-6 shift of its threshold does not flip is clear of it by that
margin, so a mismatch below is a divergence of the engine, not a tie decided by rounding.  rho is also checked on the trace.
Non-vacuity, for every case: the termination the case is named for is reached, and the oracle's run with default options
takes another trajectory (termination, iteration count or -- for the scaling and clamp cases, which change the steps but
not necessarily their number -- the trace)."""
import numpy as np
import pytest

import test_gpu_components as T
import test_gpu_lm_graphs as G
from helpers import oracle_correspond, scene
from mv_lm_icp_b200 import COST_MIXED, COST_P2P, COST_P2PLANE, PARAM_AA, PARAM_QUAT, PARAM_SE3, Engine, MvicpError, synth
from mv_lm_icp_b200.api import TERMINATION, ICP_Ceres, default_options

pytestmark = pytest.mark.gpu
COMBOS = [(PARAM_AA, COST_P2P, False), (PARAM_QUAT, COST_MIXED, True), (PARAM_SE3, COST_P2PLANE, True)]
COMBO_IDS = ["aa-p2p", "quat-mixed-robust", "se3-plane-robust"]
THRESHOLDS = ["min_relative_decrease", "function_tolerance", "parameter_tolerance", "gradient_tolerance",
              "min_trust_region_radius"]
MARGIN = 1e-6
# trace columns (oracle/oracle_icp.cpp, orc_optimize)
IT, VALID, ACC, COST, CAND, MCC, RHO, RADIUS, STEP, GRAD = range(10)


def term(name):
    return TERMINATION.index(name)


# ---- options, the bar, the guard -------------------------------------------------------------------------------------
def options(**kw):
    """(engine options, oracle options): the defaults with the given fields set to the same values on both."""
    from oracle import oracle as O
    a, b = default_options(), O.default_options()
    for k, v in kw.items():
        setattr(a, k, v); setattr(b, k, v)
    return a, b


def frame_err(P, Q):
    """max over frames of |P_f - Q_f|_max / max(1, |Q_f|_max) over the 3x4 part."""
    P = np.asarray(P)[:, :3, :]; Q = np.asarray(Q)[:, :3, :]
    return float(max(np.abs(p - q).max() / max(1.0, np.abs(q).max()) for p, q in zip(P, Q)))


def check_bar(s, P, sref, Pref, what):
    assert s["termination"] == sref["termination"], (what, s, sref)
    assert s["num_iterations"] == sref["num_iterations"], (what, s, sref)
    assert s["num_successful_steps"] == sref["num_successful_steps"], (what, s, sref)
    assert s["num_evaluations"] == 1 + sref["num_cost_evals"], (what, s, sref)
    assert s["num_linear_solves"] == sref["num_iterations"], (what, s, sref)
    for k in ("initial_cost", "final_cost"):
        assert abs(s[k] - sref[k]) <= G.COST_TOL * abs(sref[k]), (what, k, s, sref)
    err = frame_err(P, Pref)
    assert err <= G.TIGHT_TOL, (what, err)


class Problem:
    """One joint problem: frames, normals, poses, graph, fixed set and the correspondences of every edge."""

    def __init__(self, pts, nor, poses, edges, corr, w, fixed=(0,)):
        self.pts, self.nor, self.poses, self.edges, self.corr, self.w = pts, nor, np.array(poses), edges, corr, w
        self.fx = G._fixed_list(len(pts), fixed)

    def oracle(self, O, param, cost, robust, oopt):
        return O.optimize(self.pts, self.nor, self.poses, self.edges, self.corr, self.w, param=param, cost=cost,
                          robust=robust, se3_autodiff=True, threads=8, fixed=self.fx, options=oopt)


def _decisions(s, tr):
    return (s["termination"], s["num_iterations"], s["num_successful_steps"], s["num_cost_evals"],
            tuple(map(tuple, tr[:, [VALID, ACC]].astype(int))))


def guard(O, pr, param, cost, robust, oopt, sref, tr, what):
    """The decision-margin guard of the module docstring."""
    from oracle import oracle as Om
    ref = _decisions(sref, tr)
    for name in THRESHOLDS:
        v = getattr(oopt, name)
        for f in (1 - MARGIN, 1 + MARGIN):
            o2 = Om.LmOptions.from_buffer_copy(oopt)
            setattr(o2, name, v * f)
            _, s2, t2 = pr.oracle(O, param, cost, robust, o2)
            assert _decisions(s2, t2) == ref, (what, "decision within 1e-6 of", name, f)
    for r in tr[1:]:                      # rho of every step that reached the acceptance test
        if r[VALID] and r[RHO] != 0.0:
            assert abs(r[RHO] - oopt.min_relative_decrease) > MARGIN * max(abs(oopt.min_relative_decrease), 1e-300), (what, r)


def run_joint(O, pr, param, cost, robust, opts, what, eng=None, default_differs="counts"):
    """The oracle with `opts` (guarded), its default run (non-vacuity), then the engine, held to the bar.  Returns
    (engine poses, engine summary, oracle summary, oracle trace)."""
    eopt, oopt = opts
    Pref, sref, tr = pr.oracle(O, param, cost, robust, oopt)
    guard(O, pr, param, cost, robust, oopt, sref, tr, what)
    if default_differs:
        _, sd, td = pr.oracle(O, param, cost, robust, None)
        if default_differs == "counts":
            assert (sd["termination"], sd["num_iterations"]) != (sref["termination"], sref["num_iterations"]), (what, sd)
        else:
            assert td.shape != tr.shape or not np.array_equal(td, tr), what
    own = eng is None
    if own:
        eng = Engine(); eng.set_frames(pr.pts, pr.nor if all(n is not None for n in pr.nor) else None)
        eng.set_graph(pr.edges)
    eng.set_poses(pr.poses, pr.fx)
    for e, (s, _) in enumerate(pr.edges):
        if not pr.fx[s]:
            eng.set_edge(e, pr.corr[e][0], pr.corr[e][1], pr.w[e])
    s = eng.optimize(param, cost, robust, options=eopt)
    P = eng.get_poses()
    if own:
        eng.close()
    check_bar(s, P, sref, Pref, (what, param, cost, robust, TERMINATION[s["termination"]], s["num_iterations"]))
    return P, s, sref, tr


# ---- scenes ------------------------------------------------------------------------------------------------------------
def ring_problem(O, n_points, n_views=4, cfg=61):
    sc = scene(n_views, n_points, cfg)
    pts = [p.copy() for p in sc["pts"]]; nor = [n.copy() for n in sc["nor"]]
    poses = sc["poses_init"].copy()
    edges = synth.ring_edges(n_views, 2)
    corr, w = G._corr_of(oracle_correspond(O, pts, poses, edges))
    return Problem(pts, nor, poses, edges, corr, w)


def without_residuals(pr, z):
    """The problem with every correspondence of frame z removed (its edges stay, with no inlier and weight 0): z keeps its
    columns, and its block of the normal matrix is exactly zero."""
    corr, w = list(pr.corr), list(pr.w)
    for e, (s, d) in enumerate(pr.edges):
        if z in (s, d):
            corr[e] = (np.zeros(0, np.int32), np.zeros(0, np.int32)); w[e] = np.float32(0)
    out = Problem(pr.pts, pr.nor, pr.poses, pr.edges, corr, w)
    out.fx = list(pr.fx)
    return out


def moved(pr, f, t):
    """The problem with frame f translated by t (correspondences kept)."""
    out = Problem(pr.pts, pr.nor, pr.poses, pr.edges, pr.corr, pr.w)
    out.fx = list(pr.fx)
    out.poses[f][:3, 3] += t
    return out


# ---- 1. terminations on the joint path ----------------------------------------------------------------------------------
def check_max_iterations(O, n_points, param, cost, robust):
    pr = ring_problem(O, n_points)
    for k in (0, 1, 2):
        _, s, _, _ = run_joint(O, pr, param, cost, robust, options(max_num_iterations=k), ("max_iter", k))
        assert s["termination"] == term("MAX_ITERATIONS") and s["num_iterations"] == k, s
        assert s["num_linear_solves"] == k, s


def check_gradient(O, n_points, param, cost, robust):
    pr = ring_problem(O, n_points)
    _, _, tr0 = pr.oracle(O, param, cost, robust, options(max_num_iterations=0)[1])
    g0 = tr0[0, GRAD]
    _, s, _, _ = run_joint(O, pr, param, cost, robust, options(gradient_tolerance=2 * g0), "gradient at start")
    assert s["termination"] == term("GRADIENT_TOLERANCE") and s["num_iterations"] == 0, s
    assert s["initial_cost"] == s["final_cost"], s
    # after a step: the tolerance between the gradient norm at the start and at the first accepted point
    _, _, td = pr.oracle(O, param, cost, robust, None)
    acc = [i for i in range(1, len(td)) if td[i, ACC]]
    assert acc and acc[0] + 1 < len(td), td
    g1 = td[acc[0] + 1, GRAD]
    assert g1 < g0, (g0, g1)
    _, s, _, _ = run_joint(O, pr, param, cost, robust, options(gradient_tolerance=float(np.sqrt(g0 * g1))), "gradient after step")
    assert s["termination"] == term("GRADIENT_TOLERANCE") and s["num_successful_steps"] == 1, s


def check_zero_residual(O, n_points, param, cost, robust):
    """src = dst, identity matches, poses at the identity: every residual is exactly 0, so is the gradient; 0 <= 0 ends the
    solve at the start point.  (The default tolerance ends it there too: this case is about the exact zero, not a
    different trajectory, and is exempt from the non-vacuity rule.)"""
    sc = scene(2, n_points, 61)
    p = sc["pts"][1]
    idx = np.arange(len(p), dtype=np.int32)
    pr = Problem([p, p.copy()], [sc["nor"][1], sc["nor"][1].copy()], np.stack([np.eye(4)] * 2), [(1, 0)], [(idx, idx)],
                 [np.float32(0.05)])
    _, s, _, _ = run_joint(O, pr, param, cost, robust, options(gradient_tolerance=0.0), "zero residual", default_differs=None)
    assert s["termination"] == term("GRADIENT_TOLERANCE") and s["num_iterations"] == 0, s
    assert s["initial_cost"] == 0.0 and s["final_cost"] == 0.0, s


def check_min_radius(O, n_points, param, cost, robust):
    pr = ring_problem(O, n_points)
    opts = options(min_relative_decrease=10.0, function_tolerance=0.0, parameter_tolerance=0.0, min_trust_region_radius=100.0)
    P, s, sref, tr = run_joint(O, pr, param, cost, robust, opts, "min radius")
    assert s["termination"] == term("MIN_RADIUS") and s["num_successful_steps"] == 0, s
    assert s["num_iterations"] == 4, s          # 1e4 / 2 / 4 / 8 = 156 > 100, / 16 = 9.8 < 100
    assert tr[1:, VALID].all() and not tr[1:, ACC].any(), tr
    assert frame_err(P, pr.poses) <= 1e-14      # every step rejected: the start poses' parameter round trip


def turned(pr, f, deg):
    """The problem with frame f turned by `deg` degrees about a fixed oblique axis (correspondences kept)."""
    out = Problem(pr.pts, pr.nor, pr.poses, pr.edges, pr.corr, pr.w)
    out.fx = list(pr.fx)
    k = np.array([1.0, 2.0, 3.0]) / np.sqrt(14.0); th = np.radians(deg)
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(4); R[:3, :3] = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K
    out.poses[f] = R @ out.poses[f]
    return out


def check_reject_then_accept(O, n_points, param, cost, robust):
    """A frame turned far from its matches and an initial radius of 1e16: the Gauss-Newton-like first steps overshoot and are
    rejected again and again (the decrease factor doubles, the diagonal is reused) until the radius is small enough for an
    acceptance.  The first (angle, min_relative_decrease) of the list that gives two rejections followed by an acceptance is
    taken; the oracle decides it and the guard holds it clear of rounding."""
    if param == PARAM_SE3:
        pytest.skip("the SE3 parameterisation's steps are not rejected on these scenes (rho stays above 1)")
    base = ring_problem(O, n_points)
    for deg, mrd in ((90, 1e-3), (90, 0.3), (150, 1e-3), (150, 0.3)):
        pr = turned(base, 2, deg)
        opts = options(initial_trust_region_radius=1e16, min_relative_decrease=mrd)
        _, _, tr = pr.oracle(O, param, cost, robust, opts[1])
        rej = [bool(r[VALID] and not r[ACC]) for r in tr]
        if any(rej[i] and rej[i + 1] and tr[i + 2, ACC] for i in range(1, len(tr) - 2)):
            break
    else:
        pytest.fail("no (angle, min_relative_decrease) in the list gives two rejections followed by an acceptance")
    _, s, _, tr = run_joint(O, pr, param, cost, robust, opts, ("reject then accept", deg, mrd))
    i = next(i for i in range(1, len(tr) - 2) if rej[i] and rej[i + 1] and tr[i + 2, ACC])
    # the second of two rejections divides the radius by twice the factor the first one used (decrease_factor doubling)
    assert tr[i + 2, RADIUS] / tr[i + 1, RADIUS] == 0.5 * (tr[i + 1, RADIUS] / tr[i, RADIUS]), tr[i:i + 3]
    assert s["num_successful_steps"] > 0 and s["num_iterations"] > s["num_successful_steps"] + 1, s


def check_small_radius(O, n_points, param, cost, robust):
    pr = ring_problem(O, n_points)
    for r in (1e-6, 1e-5, 1e-4, 1e-3, 1e-2):
        opts = options(initial_trust_region_radius=r, max_trust_region_radius=r)
        _, sr, tr = pr.oracle(O, param, cost, robust, opts[1])
        capped = [i for i in range(1, len(tr) - 1) if tr[i, ACC] and tr[i, RHO] > 0.5 and tr[i + 1, RADIUS] == r]
        if sr["num_successful_steps"] >= 3 and capped:
            break
    else:
        pytest.fail("no radius in the list gives three accepted steps with the cap binding")
    _, s, _, tr = run_joint(O, pr, param, cost, robust, opts, ("small radius", r))
    assert (tr[:, RADIUS] <= r).all(), tr


def check_no_scaling(O, n_points, param, cost, robust):
    pr = ring_problem(O, n_points)
    run_joint(O, pr, param, cost, robust, options(jacobi_scaling=0), "no jacobi scaling", default_differs="trace")


def check_clamps(O, n_points, param, cost, robust):
    pr = ring_problem(O, n_points)
    fx = np.asarray(pr.fx, np.uint8)
    _, H, _ = O.evaluate(pr.pts, pr.nor, pr.poses, pr.edges, pr.corr, pr.w, param=param, cost=cost, robust=robust, threads=8,
                         fixed=fx)
    h = np.diag(H)
    d = h / (1 + np.sqrt(h)) ** 2                # the scaled diagonal at the start point
    mid = float(np.median(d))
    assert d.max() > mid * (1 + 1e-3) and d.min() < mid * (1 - 1e-3), d
    run_joint(O, pr, param, cost, robust, options(max_lm_diagonal=mid), "max_lm_diagonal binds", default_differs="trace")
    run_joint(O, pr, param, cost, robust, options(min_lm_diagonal=mid), "min_lm_diagonal binds", default_differs="trace")


def check_invalid_factor(O, pr, z, param, cost, robust, eng=None, tag=""):
    """min_lm_diagonal = 0 and a free frame z without residuals: its pivot is exactly 0, every step is invalid."""
    pz = without_residuals(pr, z)
    for k in (1, 5):
        P, s, _, tr = run_joint(O, pz, param, cost, robust, options(min_lm_diagonal=0.0, max_num_consecutive_invalid_steps=k),
                                ("invalid factor", z, k, tag), eng=eng)
        assert s["termination"] == term("INVALID_STEPS") and s["num_iterations"] == k, s
        assert s["num_successful_steps"] == 0 and s["num_evaluations"] == 1, s
        assert not tr[1:, VALID].any() and (tr[1:, MCC] == 0).all(), tr      # every factor failed
        if not T._nonrigid_poses(pz.poses):
            assert frame_err(P, pz.poses) <= 1e-14


def check_invalid_positions(O, n_points, param, cost, robust):
    """The zero pivot in the first free block (factored before the loop), a middle one (factored by the look-ahead, reported
    at the top of the next block step) and the last (reported after the loop)."""
    pr = ring_problem(O, n_points, n_views=5)
    for z in (1, 3, 4):
        check_invalid_factor(O, pr, z, param, cost, robust, tag=z)


def line_problem(O, n_points, thickness):
    """Two frames whose points lie on a thin cylinder around the x axis: the rotation about the axis is nearly unobservable
    (the normal matrix has a condition number ~ 1 / thickness^2)."""
    rng = np.random.default_rng(5)
    t = rng.uniform(-0.5, 0.5, n_points)
    a = rng.uniform(0, 2 * np.pi, n_points)
    p = np.stack([t, thickness * np.cos(a), thickness * np.sin(a)], 1).astype(np.float32).astype(np.float64)
    nor = np.stack([np.zeros(n_points), np.cos(a), np.sin(a)], 1).astype(np.float32).astype(np.float64)
    P1 = G._rigid(np.random.default_rng(6), 0.02, 0.01)
    idx = np.arange(n_points, dtype=np.int32)
    q = (p + rng.normal(0, 1e-3, p.shape)).astype(np.float32).astype(np.float64)    # a non-zero cost at the minimum
    return Problem([q, p], [nor, nor.copy()], np.stack([np.eye(4), P1]), [(1, 0)], [(idx, idx)], [np.float32(0.05)])


def check_model_change(O, n_points, param, cost, robust):
    """min_lm_diagonal = 0 and a radius of 1e16 on a nearly unobservable rotation: the engine's model cost change (the O(n)
    identity 1/2 (y.g~ + sum D^2 y^2)) must take the decisions the oracle takes with Ceres' -s.g~ - 1/2 s^T H~ s."""
    for th in (1e-2, 1e-3):
        pr = line_problem(O, n_points, th)
        run_joint(O, pr, param, COST_P2P, robust, options(min_lm_diagonal=0.0, initial_trust_region_radius=1e16),
                  ("model change", th), default_differs="trace")


def check_eval_failure(O, pr, param, cost, robust, f=2, eng=None, tag=""):
    """Frame f at 1e200: the squared residual overflows fp64, the start point's cost is not finite."""
    pm = moved(pr, f, [1e200, 0, 0])
    P, s, sref, _ = run_joint(O, pm, param, cost, robust, options(), ("eval failure", tag), eng=eng, default_differs=None)
    assert s["termination"] == term("EVAL_FAILURE") and s["num_iterations"] == 0 and s["num_evaluations"] == 1, s
    assert s["initial_cost"] == sref["initial_cost"] == 0.0 and s["final_cost"] == sref["final_cost"] == 0.0, (s, sref)
    if not T._nonrigid_poses(pm.poses):         # (a non-rigid pose is projected by the parameter round trip)
        assert frame_err(P, pm.poses) <= 1e-14


def check_fp32_range(O, pr, param, cost, robust, f=2, eng=None, tag=""):
    """Frame f far enough away that the cost (or, under the robust loss, a residual) exceeds FLT_MAX but stays finite in fp64."""
    pm = moved(pr, f, [1e40 if robust else 1e20, 0, 0])
    _, s, _, _ = run_joint(O, pm, param, cost, robust, options(max_num_iterations=0), ("fp32 range", tag), eng=eng)
    assert s["termination"] == term("MAX_ITERATIONS") and np.isfinite(s["initial_cost"]), s
    assert s["initial_cost"] > float(np.finfo(np.float32).max), s


@pytest.mark.parametrize("param,cost,robust", COMBOS, ids=COMBO_IDS)
@pytest.mark.parametrize("case", ["max_iterations", "gradient", "zero_residual", "min_radius", "reject_then_accept",
                                  "small_radius", "no_scaling", "clamps", "invalid_positions", "model_change"])
def test_joint_cases(oracle, case, param, cost, robust):
    globals()["check_" + case](oracle, 1500, param, cost, robust)


def test_failures_on_the_wide_graph(oracle):
    """The zero pivot in the first, a middle and the last block of a factor that lives in global memory."""
    M = 48
    edges = G.wide_graph(M)
    need, _ = G.skyline_bytes(M, edges, (0,))
    assert need > G.SMEM_LIMIT, need
    sc = scene(M, 600, 18)
    pts, nor, poses = list(sc["pts"]), list(sc["nor"]), sc["poses_init"].copy()
    corr, w = G._corr_of(oracle_correspond(oracle, pts, poses, edges))
    pr = Problem(pts, nor, poses, edges, corr, w)
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges)
    for z in (1, 24, M - 1):
        check_invalid_factor(oracle, pr, z, PARAM_SE3, COST_P2PLANE, True, eng=eng, tag=("wide", z))
    eng.close()


# ---- 2. eval paths and storage modes -------------------------------------------------------------------------------------
def check_storage_failures(O, mode, path, param, n_points):
    eng, pts, nor, poses, edges, corr, w = G._storage_setup(O, mode, path, n_points=n_points)
    pr = Problem(pts, nor, poses, edges, corr, w)
    cost = COST_P2P if mode == "f32_no_normals" else COST_P2PLANE
    for robust in (False, True):
        check_eval_failure(O, pr, param, cost, robust, eng=eng, tag=(mode, path))
        check_fp32_range(O, pr, param, cost, robust, eng=eng, tag=(mode, path))
    check_invalid_factor(O, pr, 3, param, cost, True, eng=eng, tag=(mode, path))
    eng.close()


@pytest.mark.parametrize("mode", G.MODES)
@pytest.mark.parametrize("path,param", [("unit", PARAM_AA), ("unit", PARAM_SE3), ("general", PARAM_QUAT), ("general", PARAM_SE3)])
def test_storage_modes_and_paths(oracle, mode, path, param):
    check_storage_failures(oracle, mode, path, param, 1000)


# ---- 3. component batches with mixed outcomes ----------------------------------------------------------------------------
def mixed_outcome_comps(O, n_points, nonrigid=False, wide=True):
    """A pair that converges, a component with a free frame without residuals, one with a frame at 1e200, an all-fixed
    one and (wide) the 48-view component whose factor needs global memory -- all under min_lm_diagonal = 0."""
    kw = dict(n_points=n_points, nonrigid=nonrigid)
    comps = [T.Comp(O, 2, [(1, 0), (0, 1)], cfg=11, **kw),
             T.Comp(O, 4, [(1, 0), (2, 1), (1, 2), (2, 0), (3, 0)], empty=(4,), cfg=17, **kw),
             T.Comp(O, 3, synth.ring_edges(3, 1), cfg=13, **kw),
             T.Comp(O, 3, synth.ring_edges(3, 1), fixed=(0, 1, 2), cfg=15, **kw)]
    comps[2].poses[2][:3, 3] += [1e200, 0, 0]    # after its correspondences were found
    if wide:
        comps.append(T.Comp(O, 48, G.wide_graph(48), cfg=18, n_points=600, nonrigid=nonrigid))
    return comps


EXPECT = ["?", "INVALID_STEPS", "EVAL_FAILURE", None]     # per component of mixed_outcome_comps (None: no unknowns)


def check_batch(O, comps, param, cost, robust, opts):
    """The contract of tests/test_gpu_components.py under the given (engine, oracle) options: every component of the batch
    equals a fresh engine holding only that component, bit for bit (under the same shared-settings preconditions), and is
    held to this module's bar against the oracle (with the counters, and poses per frame).  Returns (summaries, poses,
    batch)."""
    eopt, oopt = opts
    b = T.Batch(comps)
    tl = G.tile_len(b.active_slots())
    P, summ, _ = T.solve_batch(b, param, cost, robust, eopt)
    general = param != PARAM_AA and T._nonrigid_poses(b.poses)
    for k, c in enumerate(comps):
        Pk, sk = P[b.gid[k]], summ[k]
        what = (k, c.n, param, cost, robust, TERMINATION[sk["termination"]], sk["num_iterations"])
        if not c.free:
            assert np.array_equal(T._bits(Pk), T._bits(c.poses)) and sk == T.NO_UNKNOWNS, (what, sk)
            continue
        assert G.tile_len(c.active_slots()) == tl, (what, c.active_slots(), b.active_slots())
        assert (param != PARAM_AA and T._nonrigid_poses(c.poses)) == general, what
        Pf, sf, _ = T.solve_fresh(c, param, cost, robust, eopt)
        assert sk == sf, (what, sk, sf)
        assert np.array_equal(T._bits(Pk), T._bits(Pf)), what
        Pref, sref, _ = O.optimize(c.pts, c.nor, c.poses, c.edges, c.corr, c.w, param=param, cost=cost, robust=robust,
                                   se3_autodiff=True, threads=8, fixed=c.fx, options=oopt)
        check_bar(sk, Pk, sref, Pref, what)
    return summ, P, b


def check_mixed_batch(O, n_points, param, cost, robust, nonrigid=False, wide=True, max_iter=8):
    opts = options(min_lm_diagonal=0.0, max_num_iterations=max_iter)
    comps = mixed_outcome_comps(O, n_points, nonrigid, wide)
    for c in comps:
        if c.free:
            pr = Problem(c.pts, c.nor, c.poses, c.edges, c.corr, c.w); pr.fx = list(c.fx)
            _, sref, tr = pr.oracle(O, param, cost, robust, opts[1])
            guard(O, pr, param, cost, robust, opts[1], sref, tr, ("batch", c.n))
    sums, P1, b1 = check_batch(O, comps, param, cost, robust, opts)
    for k, want in enumerate(EXPECT):
        if want not in (None, "?"):
            assert sums[k]["termination"] == term(want), (k, sums[k])
    assert sums[0]["termination"] not in (term("INVALID_STEPS"), term("EVAL_FAILURE")), sums[0]
    assert all(s["num_evaluations"] <= max_iter + 2 for s in sums), sums
    # the failing components do not change the bits of the others: the batch without them gives the same bits
    good = [k for k in range(len(comps)) if k not in (1, 2)]
    b2 = T.Batch([comps[k] for k in good])
    P2, s2, _ = T.solve_batch(b2, param, cost, robust, opts[0])
    for j, k in enumerate(good):
        assert sums[k] == s2[j], (k, sums[k], s2[j])
        assert np.array_equal(T._bits(P1[b1.gid[k]]), T._bits(P2[b2.gid[j]])), k
    for k in (1, 2):
        c = comps[k]
        if not nonrigid:                  # nothing moved (a non-rigid pose is projected by the parameter round trip)
            assert frame_err(P1[b1.gid[k]], c.poses) <= 1e-14, k
    return sums


@pytest.mark.parametrize("param,cost,robust", COMBOS, ids=COMBO_IDS)
@pytest.mark.parametrize("path", ["unit", "general"])
def test_mixed_outcome_batch(oracle, param, cost, robust, path):
    if path == "general" and param == PARAM_AA:
        pytest.skip("angle-axis never takes the general frame model")
    check_mixed_batch(oracle, 1000, param, cost, robust, nonrigid=path == "general")


def test_wide_component_fails_inside_a_batch(oracle):
    """The residual-free frame inside the 48-view component of a batch: the factor in global memory fails in one CTA while
    a pair next to it converges."""
    pair = T.Comp(oracle, 2, [(1, 0), (0, 1)], cfg=11, n_points=1000)
    wide = T.Comp(oracle, 48, G.wide_graph(48), cfg=18, n_points=600, empty=[e for e, (s, d) in enumerate(G.wide_graph(48))
                                                                             if 24 in (s, d)])
    sums, _, _ = check_batch(oracle, [pair, wide], PARAM_SE3, COST_P2PLANE, True, options(min_lm_diagonal=0.0))
    assert sums[1]["termination"] == term("INVALID_STEPS") and sums[1]["num_iterations"] == 5, sums
    assert sums[0]["termination"] != term("INVALID_STEPS"), sums


# ---- 4. option rules -------------------------------------------------------------------------------------------------------
TINY = 5e-324
NAN = float("nan")


def rule_pairs():
    """(rule, {field: smallest invalid value}, {field: boundary value that is valid}) for every rule of include/mvicp.h."""
    d = default_options()
    up = lambda v: float(np.nextafter(v, np.inf))
    out = [("max_num_iterations", {"max_num_iterations": -1}, {"max_num_iterations": 0}),
           ("max_num_consecutive_invalid_steps", {"max_num_consecutive_invalid_steps": -1}, {"max_num_consecutive_invalid_steps": 0})]
    for f in ("function_tolerance", "gradient_tolerance", "parameter_tolerance", "min_relative_decrease", "min_lm_diagonal"):
        out.append((f, {f: -TINY}, {f: 0.0}))
    out += [("initial_radius>0", {"initial_trust_region_radius": 0.0, "min_trust_region_radius": TINY},
             {"initial_trust_region_radius": TINY, "min_trust_region_radius": TINY}),
            ("min_radius>0", {"min_trust_region_radius": 0.0}, {"min_trust_region_radius": TINY}),
            ("max_radius>0", {"max_trust_region_radius": 0.0, "initial_trust_region_radius": 0.0, "min_trust_region_radius": 0.0},
             {"max_trust_region_radius": TINY, "initial_trust_region_radius": TINY, "min_trust_region_radius": TINY}),
            ("min<=initial", {"min_trust_region_radius": up(d.initial_trust_region_radius)},
             {"min_trust_region_radius": d.initial_trust_region_radius}),
            ("initial<=max", {"initial_trust_region_radius": up(d.max_trust_region_radius)},
             {"initial_trust_region_radius": d.max_trust_region_radius}),
            ("max_lm_diagonal>=0", {"max_lm_diagonal": -TINY, "min_lm_diagonal": 0.0}, {"max_lm_diagonal": 0.0, "min_lm_diagonal": 0.0}),
            ("min<=max diagonal", {"min_lm_diagonal": up(d.max_lm_diagonal)}, {"min_lm_diagonal": d.max_lm_diagonal})]
    for f in ("initial_trust_region_radius", "max_trust_region_radius", "min_trust_region_radius", "min_relative_decrease",
              "min_lm_diagonal", "max_lm_diagonal", "function_tolerance", "gradient_tolerance", "parameter_tolerance"):
        out.append((f + "=nan", {f: NAN}, None))
    return out


def _opt(fields, max_iter=None):
    o = default_options()
    for k, v in fields.items():
        setattr(o, k, v)
    if max_iter is not None and "max_num_iterations" not in fields:
        o.max_num_iterations = max_iter
    return o


def check_option_rules(n_points):
    sc = scene(3, n_points, 31)
    edges = synth.ring_edges(3, 1)
    free = [0, 0, 0]
    nq = n_points * len(edges)                 # every edge searched while frame 0 is free

    def fresh():
        e = Engine(); e.set_frames(sc["pts"], sc["nor"]); e.set_graph(edges); e.set_poses(sc["poses_init"], free)
        return e

    def expect_invalid(call):
        with pytest.raises(MvicpError) as ei:
            call()
        assert ei.value.code == 1, ei.value
    ref = fresh(); ref.correspond(0.05)
    s_ref = ref.optimize(PARAM_SE3, COST_P2PLANE, True); P_ref = ref.get_poses(); ref.close()
    ref = fresh(); ref.correspond(0.05)
    c_ref = ref.optimize_components(PARAM_SE3, COST_P2PLANE, True); Pc_ref = ref.get_poses(); ref.close()
    for rule, bad, good in rule_pairs():
        o_bad = _opt(bad)
        eng = fresh(); eng.correspond(0.05)
        before = eng.get_poses()
        expect_invalid(lambda: eng.optimize(PARAM_SE3, COST_P2PLANE, True, options=o_bad))
        expect_invalid(lambda: eng.optimize_components(PARAM_SE3, COST_P2PLANE, True, options=o_bad))
        expect_invalid(lambda: eng.icp_round(0.2, PARAM_SE3, COST_P2PLANE, True, options=o_bad))
        assert np.array_equal(T._bits(eng.get_poses()), T._bits(before)), rule
        s = eng.optimize(PARAM_SE3, COST_P2PLANE, True)    # on the correspondences of correspond(0.05), not icp_round's 0.2
        assert s == s_ref and np.array_equal(T._bits(eng.get_poses()), T._bits(P_ref)), rule
        eng.close()
        eng = fresh(); eng.correspond(0.05)
        expect_invalid(lambda: eng.optimize(PARAM_SE3, COST_P2PLANE, True, options=o_bad))
        eng.correspond(0.05)
        assert eng.stats()["queries"] == nq, (rule, eng.stats())     # frame 0 is still free
        c = eng.optimize_components(PARAM_SE3, COST_P2PLANE, True)
        assert c == c_ref and np.array_equal(T._bits(eng.get_poses()), T._bits(Pc_ref)), rule
        eng.close()
        expect_invalid(lambda: ICP_Ceres._pairwise(PARAM_SE3, COST_P2P, sc["pts"][1], sc["pts"][0], options=o_bad))
        if good is None:
            continue
        o_good = _opt(good, max_iter=2)
        eng = fresh(); eng.correspond(0.05)
        eng.optimize(PARAM_SE3, COST_P2PLANE, True, options=o_good)
        eng.set_poses(sc["poses_init"], free)
        eng.optimize_components(PARAM_SE3, COST_P2PLANE, True, options=o_good)
        eng.set_poses(sc["poses_init"], free)
        eng.icp_round(0.05, PARAM_SE3, COST_P2PLANE, True, options=o_good)
        eng.close()
        ICP_Ceres._pairwise(PARAM_SE3, COST_P2P, sc["pts"][1][:200], sc["pts"][0][:200], options=o_good)


def test_option_rules():
    check_option_rules(500)
