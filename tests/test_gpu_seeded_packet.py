"""Seeded rounds before convergence (csrc/knn.cuh, knn_kernel with WW = true): each lane runs its own prologue -- start-leaf scan,
neighbour lists, stale-seed rule or greedy descent -- and the lanes the neighbour lists do not settle share one packet walk per warp.
Every case checks, round by round, that the default schedule returns bit for bit -- index and fp64 distance -- what the per-lane
search returns (MVICP_FLAG_STEP_LOOP), what the oracle's brute force returns, and what a numpy brute force in the reference's
(d0*d0 + d1*d1) + d2*d2 order with the lowest-index tie rule returns.  MVICP_FLAG_NO_OBB sends every round through knn_kernel (a
round without seeds too: greedy descent, then the walk).  The ICP cases run seeded rounds that write certificates (CERT = 1, also
with the guessed-median epilogue) followed by certified rounds, against MVICP_FLAG_NO_CERT and the step loop.  The cases take a
size scale: tests/test_hostemu_seeded_packet.py runs them small on the host model."""
import numpy as np
import pytest

from helpers import oracle_correspond, scene
from mv_lm_icp_b200 import Engine, synth
from mv_lm_icp_b200.api import FLAG_NO_ADJ, FLAG_NO_CERT, FLAG_NO_OBB, FLAG_STEP_LOOP, default_options
from test_gpu_far_packet import _f32, _numpy_nn, _pose, _sheet

pytestmark = pytest.mark.gpu


def _run(pts, edges, rounds, flags, seeds):
    eng = Engine(flags=flags)
    eng.set_frames(pts, None); eng.set_graph(edges)
    out = []
    for r, poses in enumerate(rounds):
        eng.set_poses(poses)
        if r in seeds:   # seeds written through set_edge instead of the previous round's matches
            for e, (first, second) in seeds[r].items():
                eng.set_edge(e, first, second, 1.0)
        eng.correspond(0.05)
        out.append([eng.get_nn(e) for e in range(len(edges))])
    eng.close()
    return out


def _check(O, pts, edges, rounds, flags=0, seeds=None):
    """rounds: list of pose lists; the first correspond has no seeds, every later one starts from the previous matches (or from
    seeds[r], {edge: (first, second)}, written before round r).  Frame 0 is the fixed frame, whose edges are not searched: a copy
    of the first cloud is put in front of the case's frames."""
    pts = [pts[0]] + list(pts)
    edges = [(s + 1, d + 1) for s, d in edges]
    rounds = [[np.eye(4)] + list(poses) for poses in rounds]
    seeds = {r: {e: (np.asarray(f, np.int32), np.asarray(s, np.int32)) for e, (f, s) in sd.items()} for r, sd in (seeds or {}).items()}
    got = _run(pts, edges, rounds, FLAG_NO_OBB | flags, seeds)
    lane = _run(pts, edges, rounds, FLAG_NO_OBB | FLAG_STEP_LOOP | flags, seeds)
    for r, poses in enumerate(rounds):
        ref = oracle_correspond(O, pts, poses, edges, kind="brute", fixed0=False)
        for e, (s, d) in enumerate(edges):
            i0, d0 = got[r][e]
            ni, nd = _numpy_nn(O, pts[s], pts[d], poses[s], poses[d])
            for name, (ii, dd) in (("per-lane search", lane[r][e]), ("oracle", (ref[e]["nn_idx"], ref[e]["nn_d2"])), ("numpy", (ni, nd))):
                assert np.array_equal(dd.view(np.uint64), d0.view(np.uint64)), (f"round {r} edge {e}: d2 differs from the {name}")
                assert np.array_equal(ii, i0), (f"round {r} edge {e}: {int((ii != i0).sum())} indices differ from the {name}")


def _nudged(rng, m, deg, shift):
    return [_pose(rng, deg, rng.normal(size=3) * shift) for _ in range(m)]


def case_settled_and_unsettled_mixed(O, n=6000, flags=0):
    """Sheets and volumes moved by about a leaf size: most queries stay inside their start leaf's reach, some fall through."""
    rng = np.random.default_rng(201)
    a = _sheet(rng, n); b = _sheet(rng, n + 31, tilt=-15.0)
    c = _f32(rng.uniform(-0.1, 0.1, size=(n // 2, 3)))
    edges = [(0, 1), (1, 0), (2, 0), (0, 2)]
    I = [np.eye(4)] * 3
    _check(O, [a, b, c], edges, [I, _nudged(rng, 3, 0.3, 0.002), _nudged(rng, 3, 0.6, 0.004), _nudged(rng, 3, 0.1, 0.0005)], flags)


def case_all_settled(O, n=6000):
    """The same cloud on both ends, poses standing still: every query sits on its own match, the neighbour lists settle it."""
    rng = np.random.default_rng(202)
    a = _sheet(rng, n)
    b = _f32(a[rng.permutation(n)])
    _check(O, [a, b], [(0, 1), (1, 0)], [[np.eye(4)] * 2] * 3)


def case_none_settled(O, n=6000):
    """No neighbour lists (MVICP_FLAG_NO_ADJ): every lane of every warp takes the walk."""
    case_settled_and_unsettled_mixed(O, n, flags=FLAG_NO_ADJ)


def case_stale_seeds_and_set_edge(O, n=5000):
    """Seeds far from the answer (the greedy descent after a stale start leaf) and seeds written through set_edge: random dst
    indices for part of the queries, the rest left at point 0."""
    rng = np.random.default_rng(203)
    a = _f32(rng.normal(size=(n, 3)) * 0.03)
    b = _f32(a[rng.permutation(n)][: n - 9] + rng.normal(size=(n - 9, 3)) * 0.002)
    edges = [(0, 1), (1, 0)]
    k = n // 2
    seeds = {2: {0: (rng.choice(n, k, replace=False), rng.integers(0, n - 9, k)),
                 1: (rng.choice(n - 9, k, replace=False), rng.integers(0, n, k))}}
    jump = [_pose(rng, 25, [0.05, -0.04, 0.02]), np.eye(4)]
    _check(O, [a, b], edges, [[np.eye(4)] * 2, jump, _nudged(rng, 2, 0.5, 0.003), _nudged(rng, 2, 0.5, 0.003)], seeds=seeds)


def case_ties_and_duplicates(O, n=8):
    g = np.stack(np.meshgrid(np.arange(n), np.arange(n), np.arange(max(2, n // 2))), -1).reshape(-1, 3) / 64.0
    dup = np.repeat(g, 2, axis=0)[::-1].copy()        # every point twice, in reverse order: ties resolve to the lower index
    half = g + 0.5 / 64.0                             # every query equidistant from 8 grid points
    edges = [(1, 0), (2, 0), (0, 1)]
    shift = np.eye(4); shift[:3, 3] = [1 / 128.0, 0.0, 0.0]
    back = np.eye(4); back[:3, 3] = [0.0, 1 / 128.0, 0.0]
    _check(O, [dup, half, g.copy()], edges, [[np.eye(4)] * 3, [np.eye(4), shift, np.eye(4)], [np.eye(4), back, shift]])


def case_partial_warps(O, sizes=(1, 2, 5, 7, 8, 9, 16, 31, 32, 33, 40)):
    rng = np.random.default_rng(204)
    pts = [_f32(rng.normal(size=(k, 3)) * 0.01) for k in sizes]
    m = len(pts)
    edges = [(i, (i + 1) % m) for i in range(m)] + [(i, (i + 3) % m) for i in range(m)]
    _check(O, pts, edges, [[np.eye(4)] * m, _nudged(rng, m, 3, 0.01), _nudged(rng, m, 1, 0.002)])


def case_partial_tiles(O, ks=(1, 2)):
    rng = np.random.default_rng(205)
    pts = [_f32(rng.normal(size=(1500, 3)) * 0.05)]
    for k in ks:
        for dn in (-1, 1):
            pts.append(_f32(rng.normal(size=(256 * k + dn, 3)) * 0.05))
    m = len(pts)
    edges = [(i, 0) for i in range(1, m)] + [(0, 1), (1, m - 1)]
    moved = [np.eye(4)] + _nudged(rng, m - 1, 4, 0.01)
    _check(O, pts, edges, [[np.eye(4)] * m, moved, [np.eye(4)] + _nudged(rng, m - 1, 1, 0.002)])


def case_georeferenced_fp64(O, n=4000):
    rng = np.random.default_rng(206)
    off = np.array([4.2e5, 1.3e6, 231.5])
    a = _sheet(rng, n) * 100.0 + rng.normal(size=(n, 3)) * 1e-3 + off   # not fp32-representable: fp64 records
    b = _sheet(rng, n + 5, tilt=-10.0) * 100.0 + rng.normal(size=(n + 5, 3)) * 1e-3 + off
    edges = [(0, 1), (1, 0)]
    P = np.eye(4); P[:3, 3] = [0.02, -0.01, 0.005]
    Q = np.eye(4); Q[:3, 3] = [0.021, -0.0105, 0.0049]
    _check(O, [a, b], edges, [[np.eye(4)] * 2, [P, np.eye(4)], [Q, np.eye(4)]])


CASES = [case_settled_and_unsettled_mixed, case_all_settled, case_none_settled, case_stale_seeds_and_set_edge, case_ties_and_duplicates,
         case_partial_warps, case_partial_tiles, case_georeferenced_fp64]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.__name__[5:])
def test_seeded_rounds_match_per_lane_oracle_and_numpy(oracle, case):
    case(oracle)


def icp_certified(O, n_points=5003, warm=6):
    """ICP rounds through the default schedule (far rounds, seeded rounds, a seeded round that writes certificates, certified rounds)
    against MVICP_FLAG_NO_CERT and the per-lane step loop: every round's matches and the final poses bit for bit, and the last round
    against the oracle.  Full solves, then the poses standing still (a CERT = 1 round, with or without the guessed-median epilogue,
    then certified rounds); and one LM iteration per round from the start, so that the first seeded round after the far ones runs
    the guessed-median epilogue and writes certificates (SEL + CERT)."""
    sc = scene(4, n_points, 21)
    edges = synth.ring_edges(4, 2)
    one = default_options(); one.max_num_iterations = 1
    none = default_options(); none.max_num_iterations = 0
    for warm, late in ((warm, none), (0, one)):
        engs = [Engine(flags=f) for f in (0, FLAG_NO_CERT, FLAG_STEP_LOOP)]
        for eng in engs:
            eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges); eng.set_poses(sc["poses_init"])
        for rnd in range(warm + 5):
            nn = []
            for eng in engs:
                eng.correspond(0.05)
                nn.append([eng.get_nn(e) for e in range(len(edges)) if edges[e][0] != 0])
                eng.optimize(options=None if rnd < warm else late)
            for other in nn[1:]:
                for (i0, d0), (i1, d1) in zip(nn[0], other):
                    assert np.array_equal(i0, i1) and np.array_equal(d0.view(np.uint64), d1.view(np.uint64)), rnd
        for eng in engs[1:]:
            assert np.array_equal(engs[0].get_poses(), eng.get_poses())
        st = engs[0].stats()
        assert st["cert_rounds"] >= 2 and st["select_guess_rounds"] >= 3, st
        poses = engs[0].get_poses()
        engs[0].correspond(0.05)
        ref = oracle_correspond(O, sc["pts"], poses, edges)
        for e, (s, d) in enumerate(edges):
            if s == 0:
                continue
            i, d2 = engs[0].get_nn(e)
            assert np.array_equal(i, ref[e]["nn_idx"]) and np.array_equal(d2.view(np.uint64), ref[e]["nn_d2"].view(np.uint64)), e
        for eng in engs:
            eng.close()


def test_certificates_from_the_packet_walk_keep_results(oracle):
    icp_certified(oracle)
