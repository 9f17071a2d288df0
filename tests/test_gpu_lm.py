"""GPU parity of the LM step (mvicp_optimize / mvicp_pairwise) against the CPU oracle, through the C ABI.
Bar (BASELINE.json north_star): final pose parameters within 1e-5 relative; here also equal iteration counts,
equal termination type and costs to 1e-9 relative, because both sides run the same Ceres-style state machine."""
import numpy as np
import pytest

from helpers import oracle_correspond, oracle_round, pose_rel_err, rot_err_deg, scene
from mv_lm_icp_b200 import COST_MIXED, COST_P2P, COST_P2PLANE, PARAM_AA, PARAM_QUAT, PARAM_SE3, Engine, ICP_Ceres, synth

pytestmark = pytest.mark.gpu
POSE_TOL = 1e-5      # the contract
TIGHT_TOL = 1e-8     # what identical algorithms in fp64 actually reach


def _setup(O, n_views=4, n_points=3000, cfg=7, poses_key="poses_init"):
    sc = scene(n_views, n_points, cfg)
    edges = synth.ring_edges(n_views, 2)
    ref = oracle_correspond(O, sc["pts"], sc[poses_key], edges)
    corr = [((r["first"], r["second"]) if r else (np.zeros(0, np.int32), np.zeros(0, np.int32))) for r in ref]
    weights = [np.float32(r["weight"]) if r else np.float32(0) for r in ref]
    return sc, edges, corr, weights


@pytest.mark.parametrize("param", [PARAM_AA, PARAM_QUAT, PARAM_SE3])
@pytest.mark.parametrize("cost", [COST_P2P, COST_P2PLANE, COST_MIXED])
@pytest.mark.parametrize("robust", [False, True])
def test_optimize_matches_oracle(oracle, golden_dir, param, cost, robust):
    sc, edges, corr, weights = _setup(oracle)
    eng = Engine()
    eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges); eng.set_poses(sc["poses_init"])
    for e, (f, s) in enumerate(corr):
        eng.set_edge(e, f, s, weights[e])
    summ = eng.optimize(param, cost, robust)
    P = eng.get_poses()
    Pref, sref, trace = oracle.optimize(sc["pts"], sc["nor"], sc["poses_init"], edges, corr, weights, param=param, cost=cost,
                                        robust=robust, se3_autodiff=True, threads=8)
    assert summ["termination"] == sref["termination"]
    assert summ["num_iterations"] == sref["num_iterations"]
    assert summ["num_successful_steps"] == sref["num_successful_steps"]
    assert abs(summ["initial_cost"] - sref["initial_cost"]) <= 1e-9 * sref["initial_cost"]
    assert abs(summ["final_cost"] - sref["final_cost"]) <= 1e-9 * sref["final_cost"]
    err = pose_rel_err(P, Pref)
    assert err <= POSE_TOL, err
    assert err <= TIGHT_TOL, err
    # committed golden (oracle output at generation time)
    g = np.load(f"{golden_dir}/lm_golden.npz")
    k = f"p{param}_c{cost}_r{int(robust)}"
    assert pose_rel_err(P, g[k + "_poses"]) <= POSE_TOL
    assert summ["num_iterations"] == int(g[k + "_summary"][1])
    eng.close()


def test_pipeline_round_matches_oracle(oracle):
    """correspond + optimize on the GPU vs the oracle doing both, three consecutive rounds, default flags
    (point-to-plane, SE3, robust: main_multiview.cpp:30-51)."""
    sc = scene(5, 4000, 23)
    edges = synth.ring_edges(5, 2)
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges)
    poses = sc["poses_init"].copy()
    for rnd in range(3):
        eng.set_poses(poses)
        s = eng.icp_round(0.05, PARAM_SE3, COST_P2PLANE, True)
        P = eng.get_poses()
        ref = oracle_correspond(oracle, sc["pts"], poses, edges)
        corr = [((r["first"], r["second"]) if r else (np.zeros(0, np.int32), np.zeros(0, np.int32))) for r in ref]
        w = [np.float32(r["weight"]) if r else np.float32(0) for r in ref]
        Pref, sref, _ = oracle.optimize(sc["pts"], sc["nor"], poses, edges, corr, w, param=PARAM_SE3, cost=COST_P2PLANE,
                                        robust=True, threads=8)
        assert s["num_iterations"] == sref["num_iterations"] and s["termination"] == sref["termination"]
        assert pose_rel_err(P, Pref) <= TIGHT_TOL
        poses = Pref   # both sides continue from the oracle's poses: every round has identical inputs
    eng.close()


@pytest.mark.parametrize("n_views", [29, 40])
def test_many_views_factor_in_global_memory(oracle, n_views):
    """The reference's default is --limit=40 frames (main_multiview.cpp:34): 6 x 39 = 234 unknowns.  lm_step_kernel stores the
    factor row profile by row profile (skyline), and a ring's rows span two or three pose blocks, so these factors need 17 and
    24 KB and stay in shared memory; only wide row profiles leave it (tests/test_gpu_lm_graphs.py::
    test_wide_graph_factor_in_global_memory).  Same parity bar as the small cases, two consecutive rounds."""
    sc = scene(n_views, 1500, 41)
    edges = synth.ring_edges(n_views, 2)
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges)
    poses = sc["poses_init"].copy()
    for rnd in range(2):
        eng.set_poses(poses)
        s = eng.icp_round(0.05, PARAM_SE3, COST_P2PLANE, True)
        P = eng.get_poses()
        ref = oracle_correspond(oracle, sc["pts"], poses, edges)
        corr = [((r["first"], r["second"]) if r else (np.zeros(0, np.int32), np.zeros(0, np.int32))) for r in ref]
        w = [np.float32(r["weight"]) if r else np.float32(0) for r in ref]
        Pref, sref, _ = oracle.optimize(sc["pts"], sc["nor"], poses, edges, corr, w, param=PARAM_SE3, cost=COST_P2PLANE,
                                        robust=True, threads=8)
        assert s["num_iterations"] == sref["num_iterations"] and s["termination"] == sref["termination"]
        assert pose_rel_err(P, Pref) <= TIGHT_TOL
        poses = Pref
    eng.close()


def test_converges_to_ground_truth():
    """Synthetic exactly-rigid data: 20 rounds bring every pose back to GT (the reference's visual check, README.md:156-188),
    up to the few-mm bias that matching non-overlapping regions with a 5 cm cutoff leaves (the CPU oracle ends at the same place)."""
    sc = scene(6, 20011, 22)
    frames = [__import__("mv_lm_icp_b200").Frame(p, n, P) for p, n, P in zip(sc["pts"], sc["nor"], sc["poses_init"])]
    icp = ICP_Ceres(frames)
    frames[0].fixed = True
    icp.computePoseNeighbours(2)
    e0 = max(np.linalg.norm(f.pose[:3, 3] - g[:3, 3]) for f, g in zip(frames, sc["poses_gt"]))
    for _ in range(20):
        icp.computeClosestPoints(0.05)
        icp.ceresOptimizer_sophusSE3(True, True)
    e1 = max(np.linalg.norm(f.pose[:3, 3] - g[:3, 3]) for f, g in zip(frames, sc["poses_gt"]))
    r1 = max(rot_err_deg(f.pose, g) for f, g in zip(frames, sc["poses_gt"]))
    assert e0 > 2e-2 and e1 < 5e-3 and e1 < e0 / 5 and r1 < 0.8, (e0, e1, r1)   # converges to GT up to the partial-overlap bias
    icp.engine.close()


@pytest.mark.parametrize("name,param,cost", [("pointToPoint_CeresAngleAxis", PARAM_AA, COST_P2P),
                                             ("pointToPoint_EigenQuaternion", PARAM_QUAT, COST_P2P),
                                             ("pointToPoint_SophusSE3", PARAM_SE3, COST_P2P),
                                             ("pointToPlane_CeresAngleAxis", PARAM_AA, COST_P2PLANE),
                                             ("pointToPlane_EigenQuaternion", PARAM_QUAT, COST_P2PLANE),
                                             ("pointToPlane_SophusSE3", PARAM_SE3, COST_P2PLANE)])
def test_pairwise_known_answer(oracle, golden_dir, name, param, cost):
    """main_pairwise.cpp:29-134 on the real Bunny cloud 0: dst = P * src with known 1:1 correspondences; every
    solver must recover P (README.md:141-150: diff_tra ~1e-10). Also equals the oracle's pairwise solve."""
    g = np.load(f"{golden_dir}/bunny_pair.npz")
    src, nor = g["pts0"], g["nor0"]

    def R(ax, a):
        c, s = np.cos(a), np.sin(a)
        return [np.array([[1, 0, 0], [0, c, -s], [0, s, c]]), np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]]),
                np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])][ax]
    P = np.eye(4); P[:3, :3] = R(0, np.pi / 4) @ R(1, 1.0) @ R(2, -0.2); P[:3, 3] = [0.01, -0.01, -0.005]   # main_pairwise.cpp:44-50
    dst = src @ P[:3, :3].T + P[:3, 3]; ndst = nor @ P[:3, :3].T
    fn = getattr(ICP_Ceres, name)
    Pe, s = fn(src, dst, ndst) if cost == COST_P2PLANE else fn(src, dst)
    assert np.linalg.norm(Pe[:3, 3] - P[:3, 3]) < 5e-9 and rot_err_deg(Pe, P) < 1e-5
    Po, so = oracle.pairwise(src, dst, ndst, param=param, cost=cost, se3_autodiff=False, threads=8)
    assert s["num_iterations"] == so["num_iterations"]
    assert np.max(np.abs(Pe - Po)) < 1e-8


@pytest.mark.parametrize("param", [PARAM_AA, PARAM_QUAT, PARAM_SE3])
@pytest.mark.parametrize("cost", [COST_P2P, COST_P2PLANE, COST_MIXED])
def test_real_bunny_nonrigid_poses(oracle, golden_dir, param, cost):
    """BASELINE config 1: the reference's own scans with their sample poses, which are NOT rigid (singular values
    1, 0.9957, 0.9957; SURVEY section 7).  The reference then runs its quaternion / SE3 functors on non-unit quaternions;
    the oracle restates that arithmetic and the engine's general LM path must reproduce it.  Three frames so that a
    free dst frame (s,k / k,k blocks) is exercised too: scan 0 (fixed), scan 1, and scan 0 again under a slightly
    moved copy of its (non-rigid) pose; every free frame is tied to the fixed one, so the poses are determined."""
    g = np.load(f"{golden_dir}/bunny_pair.npz")
    pts = [g["pts0"], g["pts1"], g["pts0"][::2].copy()]; nor = [g["nor0"], g["nor1"], g["nor0"][::2].copy()]
    bump = np.eye(4); bump[:3, :3] = np.array([[1, -0.004, 0.003], [0.004, 1, -0.002], [-0.003, 0.002, 1]]); bump[:3, 3] = [0.002, -0.001, 0.0015]
    poses = np.stack([g["pose0"], g["pose1"], bump @ g["pose0"]])
    edges = [(1, 0), (1, 2), (2, 1), (2, 0)]
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(edges); eng.set_poses(poses)
    eng.correspond(0.05)
    corr, w = [], []
    for e in range(len(edges)):
        f, s, d, ww = eng.get_edge(e); corr.append((f, s)); w.append(ww)
    summ = eng.optimize(param, cost, True)
    P = eng.get_poses()
    Pref, sref, _ = oracle.optimize(pts, nor, poses, edges, corr, w, param=param, cost=cost, robust=True, se3_autodiff=True, threads=8)
    assert summ["num_iterations"] == sref["num_iterations"] and summ["termination"] == sref["termination"]
    assert abs(summ["initial_cost"] - sref["initial_cost"]) <= 1e-9 * sref["initial_cost"]
    # the Eigen-quaternion parameterisation's hand-written Jacobian is not the derivative of its Plus (rotation by
    # 2|delta|, eigen_quaternion.h:89-114), so LM crawls to the iteration limit on this problem and rounding differences
    # of 1e-12 per iteration (measured: tools/dbg_general.py) grow to ~1e-6 by iteration 50; the contract is 1e-5
    tol = POSE_TOL if param == PARAM_QUAT else TIGHT_TOL
    assert abs(summ["final_cost"] - sref["final_cost"]) <= (1e-5 if param == PARAM_QUAT else 1e-9) * sref["final_cost"]
    assert pose_rel_err(P, Pref) <= tol
    # a second round continues from poses that are still non-rigid for the fixed / quaternion frames (with SE3 and
    # point-to-point the reference's renormalising Plus makes every step worse there: both sides end on the minimum
    # trust-region radius, see tools/dbg_general.py)
    eng.set_poses(Pref); eng.correspond(0.05)
    corr2, w2 = [], []
    for e in range(len(edges)):
        f, s, d, ww = eng.get_edge(e); corr2.append((f, s)); w2.append(ww)
    summ2 = eng.optimize(param, cost, True)
    P2 = eng.get_poses()
    Pref2, sref2, _ = oracle.optimize(pts, nor, Pref, edges, corr2, w2, param=param, cost=cost, robust=True, se3_autodiff=True, threads=8)
    assert summ2["num_iterations"] == sref2["num_iterations"] and summ2["termination"] == sref2["termination"]
    assert pose_rel_err(P2, Pref2) <= tol
    eng.close()


def test_full_size_round_matches_oracle(oracle):
    """BASELINE config 3 shape (20 views x 200k pts, point-to-plane, SE3, robust): one full outer round on the GPU vs the
    oracle LM on the GPU's own correspondences (their parity is covered by test_gpu_corr.py::test_full_size_properties)."""
    M, N = 20, 200_000
    sc = scene(M, N, 3)
    edges = synth.ring_edges(M, 2)
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges); eng.set_poses(sc["poses_init"])
    eng.correspond(0.05)
    corr, w = [], []
    for e, (s_, d_) in enumerate(edges):
        if s_ == 0:
            corr.append((np.zeros(0, np.int32), np.zeros(0, np.int32))); w.append(np.float32(0)); continue
        f, sec, dist, ww = eng.get_edge(e)
        corr.append((f, sec)); w.append(ww)
    summ = eng.optimize(PARAM_SE3, COST_P2PLANE, True)
    P = eng.get_poses()
    Pref, sref, _ = oracle.optimize(sc["pts"], sc["nor"], sc["poses_init"], edges, corr, w, param=PARAM_SE3, cost=COST_P2PLANE,
                                    robust=True, threads=oracle.max_threads())
    assert summ["num_iterations"] == sref["num_iterations"] and summ["termination"] == sref["termination"]
    assert abs(summ["final_cost"] - sref["final_cost"]) <= 1e-9 * sref["final_cost"]
    assert pose_rel_err(P, Pref) <= TIGHT_TOL
    eng.close()


def test_frame0_is_fixed_inside_the_optimiser():
    """Every ceresOptimizer* sets frames[0]->fixed itself (icp-ceres.cpp:242-244,342-344,417-419) and works whether or not the
    caller had set it before computeClosestPoints (ADVICE round 1): same poses either way, and the pose graph built after a
    solve sees the optimised poses."""
    import mv_lm_icp_b200 as mv
    sc = scene(4, 3000, 7)
    out = []
    for pre_fixed in (True, False):
        frames = [mv.Frame(p, n, P) for p, n, P in zip(sc["pts"], sc["nor"], sc["poses_init"])]
        icp = ICP_Ceres(frames)
        frames[0].fixed = pre_fixed
        icp.computePoseNeighbours(2)
        for _ in range(2):
            icp.computeClosestPoints(0.05)
            icp.ceresOptimizer_sophusSE3(True, True)
        assert frames[0].fixed
        out.append(np.stack([f.pose for f in frames]))
        g = icp.engine.pose_graph_knn(2)     # from the CURRENT poses: the engine's host mirror follows the solve
        d = np.linalg.norm(out[-1][:, None, :3, 3] - out[-1][None, :, :3, 3], axis=2).astype(np.float32)
        for i in range(4):
            want = sorted((d[i, j], j) for j in range(4) if j != i)[:2]
            assert [b for a, b in g if a == i] == [j for _, j in want]
        icp.engine.close()
    assert np.max(np.abs(out[0][0] - sc["poses_init"][0])) < 1e-14   # frame 0 only goes through the parameter round trip (icp-ceres.cpp:472-474)
    assert np.max(np.abs(out[0] - out[1])) < 1e-12


def _eigen_rotation_of(q):
    """Quaterniond::toRotationMatrix without normalisation (what eigenQuaternionToIso applies, icp-ceres.cpp:117-122)."""
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def test_quaternion_parameterisation_drifts_off_the_unit_sphere(oracle):
    """Every solve writes quaternion -> matrix back without normalising and the next one reads it with Quaterniond(matrix): with
    the Eigen-quaternion parameterisation |q|^2 - 1 grows by a constant factor per round (measured 1.3x here, faster on the 40-view
    scene: the 20-round config-4 run crossed the 1e-9 that the unit-quaternion LM path assumes in round 15 and stopped with
    MVICP_ERR_NONRIGID).  The reference just keeps going on non-unit quaternions, so the engine has to notice the drift ON ITS
    OWN poses -- no mvicp_set_poses in between -- and switch to the general frame model.  Start just below the threshold."""
    from scipy.spatial.transform import Rotation as Rot
    sc = scene(6, 3000, 7)
    edges = synth.ring_edges(6, 2)
    P0 = sc["poses_init"].copy()
    for i in range(1, 6):
        P0[i][:3, :3] = _eigen_rotation_of(Rot.from_matrix(P0[i][:3, :3]).as_quat() * np.sqrt(1 + 7e-10))
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges); eng.set_poses(P0)
    poses, cache, errs = P0.copy(), {}, []
    for rnd in range(8):
        s = eng.icp_round(0.05, PARAM_QUAT, COST_MIXED, True)
        poses, sref, _ = oracle_round(oracle, sc["pts"], sc["nor"], poses, edges, PARAM_QUAT, COST_MIXED, index_cache=cache)
        assert s["num_iterations"] == sref["num_iterations"], rnd
        errs.append(pose_rel_err(eng.get_poses(), poses))
    P = eng.get_poses()
    assert max(np.abs(P[i][:3, :3].T @ P[i][:3, :3] - np.eye(3)).max() for i in range(6)) > 4e-9     # well off the sphere by now
    assert max(errs) <= POSE_TOL, errs
    assert errs[-1] <= 1e-11, errs      # only the general frame model follows the reference's non-unit arithmetic this closely
    eng.close()
