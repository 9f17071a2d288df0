"""Seeded fuzzing of the correspondence step against the oracle: random cloud shapes (surface, quantised grid with exact
distance ties, collinear, identical points, tiny clouds), coordinate scales and offsets (stress for the fp32 screening bound),
georeferenced scans (metres at a 1e5-1e6 offset, fp64 storage), rigid and non-rigid poses, cutoffs, every NN schedule, several
seeded rounds; the converged-round shortcuts; the LM step.  The case functions run on whichever library mv_lm_icp_b200._lib
has bound: run as a script, this file binds the host model of the engine (tools/hostemu); tests/test_gpu_fuzz.py runs the
same seeds on the GPU.
usage: python tools/fuzz_hostemu.py [n_cases] [first_seed]"""
import ctypes as C, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from mv_lm_icp_b200 import _lib, Engine
from oracle import oracle as O
from helpers import oracle_correspond


def rot(rng, s):
    w = rng.normal(0, s, 3); th = np.linalg.norm(w) + 1e-300; k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def cloud(rng, kind, n, scale, offset):
    if kind == 0:      # wavy surface
        x, y = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n); p = np.stack([x, y, 0.2 * np.sin(3 * x) * np.cos(2 * y) + 1e-3 * rng.normal(size=n)], 1)
    elif kind == 1:    # quantised grid: masses of exact ties
        p = np.round(rng.uniform(-1, 1, (n, 3)) * 8) / 8
    elif kind == 2:    # collinear
        p = np.outer(rng.uniform(-1, 1, n), [1.0, 0.5, -0.25])
    elif kind == 3:    # all identical
        p = np.tile(rng.uniform(-1, 1, 3), (n, 1))
    else:              # gaussian blob
        p = rng.normal(size=(n, 3))
    return p * scale + offset


def brute_nn(dst, q):
    """Exact nearest neighbour of every query by brute force: (d0*d0 + d1*d1) + d2*d2 in fp64, ties to the lowest index."""
    idx = np.empty(len(q), np.int32); d2 = np.empty(len(q))
    for a in range(0, len(q), 256):
        d = q[a:a + 256, None, :] - dst[None, :, :]
        D = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        j = np.argmin(D, 1)
        idx[a:a + 256] = j; d2[a:a + 256] = D[np.arange(len(j)), j]
    return idx, d2


def one_case(seed):
    """The random scene of one(seed): clouds, edges, cutoff, NN schedule and the poses of three seeded rounds."""
    rng = np.random.default_rng(seed)
    M = int(rng.integers(2, 5))
    scale = float(rng.choice([1e-3, 1.0, 1e3])); offset = rng.normal(0, 1, 3) * scale * float(rng.choice([0, 1, 100]))
    f32 = bool(rng.integers(0, 2))
    pts = []
    for v in range(M):
        n = int(rng.choice([1, 2, 7, 8, 9, 33, 500, 3000]))
        p = cloud(rng, int(rng.integers(0, 5)), n, scale, offset)
        pts.append(p.astype(np.float32).astype(np.float64) if f32 else p)
    poses = []
    for v in range(M):
        P = np.eye(4); P[:3, :3] = rot(rng, 0.3); P[:3, 3] = rng.normal(0, 0.2, 3) * scale
        if rng.integers(0, 3) == 0:
            P[:3, :3] = P[:3, :3] @ np.diag(1 + rng.normal(0, 1e-3, 3))      # not a rotation
        poses.append(P)
    edges = [(s, d) for s in range(M) for d in range(M) if s != d and rng.integers(0, 2)] or [(1, 0)]
    thresh = float(rng.choice([0.05, 0.5, 5.0])) * scale
    flags = int(rng.choice([0, 1, 4, 8, 12, 16, 17, 24]))
    rounds = []
    for rnd in range(3):
        P = [p.copy() for p in poses]
        for v in range(1, M):
            P[v][:3, 3] += rng.normal(0, [0.1, 1e-3, 1e-5][rnd], 3) * scale
        rounds.append(P)
    return dict(name=("one", seed), pts=pts, edges=edges, thresh=thresh, flags=flags, rounds=rounds)


def geo_case(seed):
    """Georeferenced scans: clouds 1-10 m across at an offset of 1e5-1e6 m, stored in fp64.  There neighbouring fp32 values are
    up to 0.06 m apart -- coarser than the points -- so fp32 screen coordinates and tree-sort keys collide, and the screen's error
    allowance is metres wide.  Poses rotate about the scan's centre; three seeded rounds, as in one_case."""
    rng = np.random.default_rng(90_000 + seed)
    M = int(rng.integers(2, 5))
    extent = float(rng.uniform(1, 10)); centre = rng.uniform(1e5, 1e6, 3) * rng.choice([-1.0, 1.0], 3)
    pts = [cloud(rng, int(rng.integers(0, 5)), int(rng.choice([1, 9, 33, 500, 3000])), 0.5 * extent, centre) for v in range(M)]
    poses = []
    for v in range(M):
        R = rot(rng, float(rng.choice([0.3, 0.01])))
        P = np.eye(4); P[:3, :3] = R; P[:3, 3] = centre - R @ centre + rng.normal(0, 0.05, 3) * extent
        poses.append(P)
    edges = [(s, d) for s in range(M) for d in range(M) if s != d and rng.integers(0, 2)] or [(1, 0)]
    thresh = float(rng.choice([0.01, 0.1, 1.0])) * extent
    flags = int(rng.choice([0, 1, 4, 8, 12, 16, 17, 24]))
    rounds = []
    for rnd in range(3):
        P = [p.copy() for p in poses]
        for v in range(1, M):
            P[v][:3, 3] += rng.normal(0, [0.1, 1e-3, 1e-5][rnd], 3) * extent
        rounds.append(P)
    return dict(name=("geo", seed), pts=pts, edges=edges, thresh=thresh, flags=flags, rounds=rounds)


def run_case(case, extra_flags=0, brute=False):
    """Runs the rounds of a case (one_case / geo_case) under its schedule | extra_flags and checks every round against the
    oracle bit for bit -- matches, distances, inlier lists, weight -- and, with brute=True, the first round against brute_nn
    over the oracle's query points.  Returns the matches [round][edge] = (index, d2) of the edges that have a result."""
    pts, edges, thresh, tag = case["pts"], case["edges"], case["thresh"], case["name"]
    M = len(pts)
    eng = Engine(flags=case["flags"] | extra_flags); eng.set_frames(pts, None); eng.set_graph(edges)
    fixed = [1] + [0] * (M - 1)
    out = []
    for rnd, P in enumerate(case["rounds"]):
        eng.set_poses(P, fixed); eng.correspond(thresh)
        ref = oracle_correspond(O, pts, P, edges, thresh=np.float32(thresh), threads=4)
        nn = []
        for e, r in enumerate(ref):
            if r is None:
                continue
            i, d2 = eng.get_nn(e)
            if brute and rnd == 0:
                s, d = edges[e]
                bi, bd = brute_nn(pts[d], O.edge_queries(pts[s], P[s], P[d]))
                assert np.array_equal(bd.view(np.uint64), r["nn_d2"].view(np.uint64)) and np.array_equal(bi, r["nn_idx"]), (tag, e, "oracle vs brute force")
            assert np.array_equal(d2.view(np.uint64), r["nn_d2"].view(np.uint64)), (tag, rnd, e, "d2")
            assert np.array_equal(i, r["nn_idx"]), (tag, rnd, e, "idx", int(np.sum(i != r["nn_idx"])))
            f, s, dist, w = eng.get_edge(e)
            assert np.array_equal(f, r["first"]) and np.array_equal(s, r["second"]), (tag, rnd, e, "inliers")
            if len(f):
                assert np.float32(w).view(np.uint32) == np.float32(r["weight"]).view(np.uint32), (tag, rnd, e, "weight", w, r["weight"])
            nn.append((i, d2))
        out.append(nn)
    eng.close()
    return out


def one(seed):
    c = one_case(seed)
    run_case(c)
    return len(c["pts"]), c["flags"]


def one_geo(seed):
    c = geo_case(seed)
    run_case(c)
    return len(c["pts"]), c["flags"], [len(p) for p in c["pts"]]


def one_steady(seed):
    """Converged-round shortcuts (guessed median select, certified matches) on the random shapes of one(): rounds whose previous
    solve took 0 or 1 LM iterations, compared bit for bit with an engine that has both shortcuts switched off, and with the oracle
    at the end.  Degenerate clouds (exact ties, duplicates, single points) must never certify a wrong match."""
    from mv_lm_icp_b200.api import FLAG_NO_CERT, FLAG_NO_SELECT_GUESS, default_options
    rng = np.random.default_rng(50_000 + seed)
    M = int(rng.integers(2, 5))
    scale = float(rng.choice([1e-3, 1.0, 1e3])); offset = rng.normal(0, 1, 3) * scale * float(rng.choice([0, 1, 100]))
    f32 = bool(rng.integers(0, 2))
    pts = []
    for v in range(M):
        n = int(rng.choice([1, 2, 7, 8, 9, 33, 500, 3000]))
        p = cloud(rng, int(rng.integers(0, 5)), n, scale, offset)
        pts.append(p.astype(np.float32).astype(np.float64) if f32 else p)
    poses = []
    for v in range(M):
        P = np.eye(4); P[:3, :3] = rot(rng, 0.02); P[:3, 3] = rng.normal(0, 0.01, 3) * scale
        poses.append(P)
    poses[0] = np.eye(4)
    edges = [(s, d) for s in range(M) for d in range(M) if s != d and rng.integers(0, 2)] or [(1, 0)]
    thresh = float(rng.choice([0.05, 0.5, 5.0])) * scale
    base = int(rng.choice([0, 4, 8, 16]))
    engs = [Engine(flags=base), Engine(flags=base | FLAG_NO_CERT | FLAG_NO_SELECT_GUESS)]
    opts = []
    for it in (0, 1, 1, 0, 1, 1):
        o = default_options(); o.max_num_iterations = it; opts.append(o)
    for eng in engs:
        eng.set_frames(pts, None); eng.set_graph(edges); eng.set_poses(poses)
    for rnd, o in enumerate(opts):
        out = []
        for eng in engs:
            eng.correspond(thresh)
            out.append(([eng.get_nn(e) for e in range(len(edges)) if edges[e][0] != 0], [eng.get_edge(e, arrays=False) for e in range(len(edges))]))
            try:
                eng.optimize(cost=0, options=o)
            except Exception as ex:      # a degenerate system may be rejected; both engines must then agree on that too
                out[-1] = out[-1] + (str(ex),)
        assert len(out[0]) == len(out[1]), (seed, rnd, out[0][2:], out[1][2:])
        for (i0, d0), (i1, d1) in zip(out[0][0], out[1][0]):
            assert np.array_equal(i0, i1) and np.array_equal(d0.view(np.uint64), d1.view(np.uint64)), (seed, rnd, "nn")
        assert out[0][1] == out[1][1], (seed, rnd, "count / weight")
        assert np.array_equal(np.asarray(engs[0].get_poses()).view(np.uint64), np.asarray(engs[1].get_poses()).view(np.uint64)), (seed, rnd, "poses")
    P = engs[0].get_poses()
    if np.all(np.isfinite(P)):
        engs[0].correspond(thresh)
        ref = oracle_correspond(O, pts, P, edges, thresh=np.float32(thresh), threads=4)
        for e, r in enumerate(ref):
            if r is None:
                continue
            i, d2 = engs[0].get_nn(e)
            assert np.array_equal(d2.view(np.uint64), r["nn_d2"].view(np.uint64)) and np.array_equal(i, r["nn_idx"]), (seed, e, "oracle")
    st = engs[0].stats()
    for eng in engs:
        eng.close()
    return M, base, st["select_guess_rounds"], st["cert_rounds"], st["cert_reused"]


def one_lm(seed):
    """LM step on a well-posed random scene: same termination, iteration counts and poses (1e-8) as the oracle."""
    from mv_lm_icp_b200 import synth
    from helpers import pose_rel_err
    rng = np.random.default_rng(10_000 + seed)
    M = int(rng.integers(2, 7)); n = int(rng.choice([300, 1000, 2500]))
    sc = synth.make_scene(M, n, config_id=100 + seed)
    edges = synth.ring_edges(M, int(rng.integers(1, 3))) if M > 2 else [(1, 0), (0, 1)]
    param, cost, robust = int(rng.integers(0, 3)), int(rng.integers(0, 3)), bool(rng.integers(0, 2))
    poses = sc["poses_init"].copy()
    if rng.integers(0, 3) == 0 and param != 0:
        poses[1][:3, :3] = poses[1][:3, :3] @ np.diag(1 + rng.normal(0, 1e-3, 3))     # general (non-unit quaternion) path
    ref = oracle_correspond(O, sc["pts"], poses, edges)
    corr = [((r["first"], r["second"]) if r else (np.zeros(0, np.int32), np.zeros(0, np.int32))) for r in ref]
    w = [np.float32(r["weight"]) if r else np.float32(0) for r in ref]
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges); eng.set_poses(poses)
    for e, (f, s2) in enumerate(corr):
        eng.set_edge(e, f, s2, w[e])
    summ = eng.optimize(param, cost, robust); P = eng.get_poses(); eng.close()
    Pref, sref, _ = O.optimize(sc["pts"], sc["nor"], poses, edges, corr, w, param=param, cost=cost, robust=robust, se3_autodiff=True, threads=4)
    assert summ["termination"] == sref["termination"] and summ["num_iterations"] == sref["num_iterations"], (seed, summ, sref)
    err = pose_rel_err(P, Pref)
    assert err <= 1e-8, (seed, err, param, cost, robust)
    return M, n, param, cost, robust, summ["num_iterations"]


if __name__ == "__main__":
    sys.path.insert(0, os.path.join(ROOT, "tools", "hostemu"))
    import build_hostemu
    lib = C.CDLL(build_hostemu.build()); lib.mvicp_last_error.restype = C.c_char_p; _lib._lib = lib
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 50; s0 = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    for seed in range(s0, s0 + n):
        info = one(seed)
        print("seed", seed, "ok", info, flush=True)
        if seed % 4 == 0:
            print("seed", seed, "lm ok", one_lm(seed), flush=True)
        if seed % 2 == 0:
            print("seed", seed, "steady ok", one_steady(seed), flush=True)
        if seed % 4 == 1:
            print("seed", seed, "geo ok", one_geo(seed), flush=True)
