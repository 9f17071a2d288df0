"""Regenerates tests/golden/*.npz.  Run in the build container (needs /root/reference):  python tests/golden/make_golden.py

bunny_pair.npz   config 1 of BASELINE.json: the reference's own sample scans samples/Bunny_RealData/cloudXYZ_{0,1}.xyz
                 (x y z nx ny nz per line; the loader's trailing garbage point, common.h:224-239, is NOT reproduced)
                 with poses_{0,1}.txt (4x4 row-major).  Stored as float64 exactly as parsed.
                 + nn_idx / nn_d2: output of the REFERENCE's nanoflann (oracle/_ref/libref_nanoflann.so, compiled from
                 /root/reference/include/nanoflann.hpp) for edge 1 -> 0 under those poses, i.e. the pinned answer of
                 Frame::computeClosestPointsToNeighbours' inner loop (frame.cpp:129-138);
                 + first/second/dist/weight of frame.cpp:140-176 from those.
dino_pair.npz    the reference's second sample set, samples/dinosaur/cloud_{1,2}.xyz with pose_{1,2}.txt: millimetre units
                 (|coordinates| up to 686, NN distances of tens of mm), 5-digit pose matrices (not exactly orthonormal):
                 edge 2 -> 1, reference nanoflann answer + frame.cpp:140-176 at cutoff 25 (the default 0.05 m is meaningless
                 in mm); pins the fp32 screening bound at a different coordinate magnitude.
lm_golden.npz    oracle LM outputs (final poses, iteration trace) on a small seeded synthetic scene for every
                 parameterisation x cost; pins the oracle against accidental change (NOT against Ceres: unpinned).
bunny18.npz      the reference's DEFAULT multiview workload (main_multiview.cpp:33-36,63: --limit=40 --step=2 on Bunny_RealData): the 18
                 scans cloudXYZ_{0,2,..,34}.xyz (224 673 points; xyz only -- the default run recomputes the normals; stored as int32
                 units of 1e-8 m, which is lossless for the <= 8-decimal text: parsed double == int / 1e8 exactly) with poses_{0,2,..,34}.txt
                 (ground truth, non-rigid: singular values 1, 0.9957, 0.9957) and the initial poses of main_multiview.cpp:78-84
                 (frame 0 = GT, the others addNoise(GT, 0.02, 0.01), common.h:38-67; the reference's default-seeded mt19937 stream
                 is not reproduced -- same noise model, numpy seed 0xB18).  Used by `bench.py --config real` and tests/test_gpu_real18.py.
sophus_vectors.npz  the SE3 group elements / tangents of ext/sophus-ceres/test/core/test_se3.cpp:40-82 (values only).
ref_nanoflann.npz   answers of the reference's nanoflann for tests/test_oracle_corr.py (a synthetic edge as sha256, k-NN on bunny_pair).
functor_pin.npz     outputs of the reference's cost-functor text on the first inputs of tests/test_oracle_functor_pin.py.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402
from mv_lm_icp_b200 import synth  # noqa: E402

REF = "/root/reference/samples/Bunny_RealData"
OUT = os.path.dirname(os.path.abspath(__file__))


def bunny_pair():
    c = [np.loadtxt(f"{REF}/cloudXYZ_{i}.xyz") for i in (0, 1)]
    P = [np.loadtxt(f"{REF}/poses_{i}.txt") for i in (0, 1)]
    ref = O.KdIndex(c[0][:, :3], "ref")
    idx, d2 = ref.closest_points(c[1][:, :3], P[1], P[0])
    first, second, dist, w, med = O.filter_edge(idx, d2, np.float32(0.05))
    np.savez_compressed(os.path.join(OUT, "bunny_pair.npz"), pts0=c[0][:, :3], nor0=c[0][:, 3:6], pts1=c[1][:, :3],
                        nor1=c[1][:, 3:6], pose0=P[0], pose1=P[1], nn_idx=idx, nn_d2=d2, first=first, second=second,
                        dist=dist, weight=w, median=med)
    print("bunny_pair:", c[0].shape, c[1].shape, "inliers", len(first), "weight", w)


def dino_pair():
    D = "/root/reference/samples/dinosaur"
    c = [np.loadtxt(f"{D}/cloud_{i}.xyz") for i in (1, 2)]
    P = [np.loadtxt(f"{D}/pose_{i}.txt") for i in (1, 2)]
    ref = O.KdIndex(c[0][:, :3], "ref")
    idx, d2 = ref.closest_points(c[1][:, :3], P[1], P[0])
    first, second, dist, w, med = O.filter_edge(idx, d2, np.float32(25.0))
    np.savez_compressed(os.path.join(OUT, "dino_pair.npz"), pts0=c[0][:, :3], nor0=c[0][:, 3:6], pts1=c[1][:, :3], nor1=c[1][:, 3:6],
                        pose0=P[0], pose1=P[1], nn_idx=idx, nn_d2=d2, first=first, second=second, dist=dist, weight=w, median=med)
    print("dino_pair:", c[0].shape, c[1].shape, "inliers", len(first), "weight", w)


def bunny18():
    ids = list(range(0, 36, 2))
    xyz, off, gt, init = [], [0], [], []
    rng = np.random.default_rng(0xB18)
    for k, i in enumerate(ids):
        c = np.loadtxt(f"{REF}/cloudXYZ_{i}.xyz")[:, :3]
        um = np.rint(c * 1e8).astype(np.int64)
        assert np.abs(um).max() < 2 ** 31 and np.array_equal(um.astype(np.float64) / 1e8, c), "int32 x 1e-8 m must be lossless"
        xyz.append(um.astype(np.int32)); off.append(off[-1] + len(c))
        P = np.loadtxt(f"{REF}/poses_{i}.txt")
        gt.append(P)
        Q = P.copy()
        if k > 0:   # addNoise (common.h:38-67): pose * SO3::exp(sigma w), translation += sigmat t
            Q[:3, :3] = P[:3, :3] @ synth._so3_exp(rng.normal(0.0, 1.0, 3) * 0.02)
            Q[:3, 3] = P[:3, 3] + rng.normal(0.0, 1.0, 3) * 0.01
        init.append(Q)
    np.savez_compressed(os.path.join(OUT, "bunny18.npz"), n_frames=len(ids), frame_ids=np.array(ids), offsets=np.array(off, np.int64),
                        xyz_e8=np.concatenate(xyz), poses_gt=np.stack(gt), poses_init=np.stack(init))
    print("bunny18:", off[-1], "points", os.path.getsize(os.path.join(OUT, "bunny18.npz")) / 1e6, "MB")


def lm_golden():
    sc = synth.make_scene(4, 3000, config_id=7)
    edges = synth.ring_edges(4, 2)
    idxs = [O.KdIndex(p, "kd") for p in sc["pts"]]
    corr, weights = [], []
    for s, d in edges:
        i, d2 = idxs[d].closest_points(sc["pts"][s], sc["poses_init"][s], sc["poses_init"][d])
        f, sec, dist, w, _ = O.filter_edge(i, d2, np.float32(0.05))
        corr.append((f, sec)); weights.append(w)
    out = {}
    for param in (0, 1, 2):
        for cost in (0, 1, 2):
            for robust in (0, 1):
                P, s, tr = O.optimize(sc["pts"], sc["nor"], sc["poses_init"], edges, corr, weights, param=param, cost=cost,
                                      robust=bool(robust), se3_autodiff=True, threads=1)
                k = f"p{param}_c{cost}_r{robust}"
                out[k + "_poses"] = P; out[k + "_trace"] = tr
                out[k + "_summary"] = np.array([s["termination"], s["num_iterations"], s["num_successful_steps"]], np.int64)
                out[k + "_cost"] = np.array([s["initial_cost"], s["final_cost"]])
                print(k, O.TERMINATION[s["termination"]], s["num_iterations"], s["initial_cost"], s["final_cost"])
    np.savez_compressed(os.path.join(OUT, "lm_golden.npz"), **out)


def ref_nanoflann():
    """Answers of the reference's nanoflann for tests/test_oracle_corr.py: sha256 of the 1-NN indices / squared distances of the
    synthetic edge of test_restatement_equals_reference_nanoflann, and the 10-NN of every 53rd point of bunny_pair's pts0."""
    import hashlib
    sys.path.insert(0, os.path.dirname(OUT))
    from helpers import scene
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
    sc = scene(3, 20000, 32)
    out = {}
    for k, poses in enumerate((sc["poses_init"], sc["poses_gt"])):
        idx, d2 = O.KdIndex(sc["pts"][0], "ref").closest_points(sc["pts"][1], poses[1], poses[0], threads=4)
        out[f"synth_idx_sha{k}"] = np.array(sha(idx)); out[f"synth_d2_sha{k}"] = np.array(sha(d2))
    pts = np.load(os.path.join(OUT, "bunny_pair.npz"))["pts0"]
    rf = O.KdIndex(pts, "ref")
    nn = [O.knn(rf, pts[i], 10) for i in range(0, len(pts), 53)]
    out["bunny_knn_idx"] = np.stack([a for a, _ in nn]); out["bunny_knn_d2"] = np.stack([b for _, b in nn])
    np.savez_compressed(os.path.join(OUT, "ref_nanoflann.npz"), **out)


def functor_pin(n_global=32, n_pairwise=16, n_quat=100):
    """Outputs of the reference's functor text (oracle/_ref/libref_functors.so) on the first inputs of every case of
    tests/test_oracle_functor_pin.py."""
    import ctypes as C
    sys.path.insert(0, os.path.dirname(OUT))
    import test_oracle_functor_pin as T
    out = {}
    for param in (0, 1, 2):
        for plane in (0, 1):
            res = [O.functor_eval(param, plane, *a, "ref") for a, _ in zip(T._global_cases(param, plane), range(n_global))]
            out[f"global_{param}{plane}_r"] = np.stack([r for r, _ in res]); out[f"global_{param}{plane}_j"] = np.stack([j for _, j in res])
            res = [O.functor_eval_pairwise_ref(param, plane, *a) for a, _ in zip(T._pairwise_cases(param, plane), range(n_pairwise))]
            out[f"pairwise_{param}{plane}_r"] = np.stack([r for r, _ in res]); out[f"pairwise_{param}{plane}_j"] = np.stack([j for _, j in res])
    lib = O.ref_functors()
    P = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    qr, qj = [], []
    for (x, d), _ in zip(T._quat_cases(), range(n_quat)):
        o = np.zeros(4); lib.ref_quat_plus(P(x), P(d), P(o)); j = np.zeros(12); lib.ref_quat_jacobian(P(x), P(j))
        qr.append(o); qj.append(j)
    out["quat_r"] = np.stack(qr); out["quat_j"] = np.stack(qj)
    np.savez_compressed(os.path.join(OUT, "functor_pin.npz"), **out)


def sophus_vectors():
    # ext/sophus-ceres/test/core/test_se3.cpp:40-65: SE3(SO3::exp(w), t) ; :67-82 tangents (upsilon, omega)
    pi = np.pi
    el = [([0.2, 0.5, 0.0], [0, 0, 0]), ([0.2, 0.5, -1.0], [10, 0, 0]), ([0.0, 0.0, 0.0], [0, 100, 5]),
          ([0.0, 0.0, 0.00001], [0, 0, 0]), ([0.0, 0.0, 0.00001], [0, -0.00000001, 0.0000000001]),
          ([0.0, 0.0, 0.00001], [0.01, 0, 0]), ([pi, 0, 0], [4, -5, 0]),
          ([0.2, 0.5, 0.0], [0, 0, 0]), ([0.3, 0.5, 0.1], [2, 0, -7])]
    tg = [[0, 0, 0, 0, 0, 0], [1, 0, 0, 0, 0, 0], [0, 1, 0, 1, 0, 0], [0, -5, 10, 0, 0, 0], [-1, 1, 0, 0, 0, 1],
          [20, -1, 0, -1, 1, 0], [30, 5, -1, 20, -1, 0]]
    np.savez_compressed(os.path.join(OUT, "sophus_vectors.npz"), so3_omega=np.array([e[0] for e in el], float),
                        trans=np.array([e[1] for e in el], float), tangents=np.array(tg, float))


if __name__ == "__main__":
    only = sys.argv[1:]
    for fn in (bunny_pair, dino_pair, lm_golden, sophus_vectors, bunny18, ref_nanoflann, functor_pin):
        if not only or fn.__name__ in only:
            fn()
