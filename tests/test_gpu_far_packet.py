"""The far rounds' packet walk (csrc/far.cuh, knn_far_kernel): the 32 queries of a warp share one depth-first walk of the dst tree.
Every case targets a place where a warp's queries are NOT coherent or the warp is NOT full, and checks, for a round without seeds
and a round with stale seeds (both far rounds), that the default engine returns bit for bit -- index and fp64 distance -- what the
per-lane search returns (MVICP_FLAG_NO_OBB: every round runs knn_kernel), what the oracle's brute force returns, and what a numpy
brute force in the reference's (d0*d0 + d1*d1) + d2*d2 order with the lowest-index tie rule returns.  The cases take a size scale:
tests/test_hostemu_far_packet.py runs them small on the host model."""
import numpy as np
import pytest

from helpers import oracle_correspond
from mv_lm_icp_b200 import Engine
from mv_lm_icp_b200.api import FLAG_NO_OBB

pytestmark = pytest.mark.gpu


def _rot(rng, deg):
    a = rng.normal(size=3); a /= np.linalg.norm(a)
    t = np.deg2rad(deg)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(t) * K + (1 - np.cos(t)) * K @ K


def _pose(rng, deg, shift):
    P = np.eye(4); P[:3, :3] = _rot(rng, deg); P[:3, 3] = shift
    return P


def _f32(x):
    return np.asarray(x, np.float32).astype(np.float64)


def _numpy_nn(O, src, dst, Ps, Pd):
    q = O.edge_queries(src, Ps, Pd)
    idx = np.empty(len(q), np.int32); best = np.empty(len(q))
    for a in range(0, len(q), 512):
        d = q[a:a + 512, None, :] - dst[None, :, :]
        d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        i = np.argmin(d2, axis=1)                    # first occurrence: the lowest index among exact ties
        idx[a:a + 512] = i; best[a:a + 512] = d2[np.arange(len(i)), i]
    return idx, best


def _check(O, pts, edges, rounds):
    """rounds: list of pose lists; the first correspond has no seeds, the next ones start from the previous matches.  Frame 0 is
    the fixed frame, whose edges are not searched: a copy of the first cloud is put in front of the case's frames."""
    pts = [pts[0]] + list(pts)
    edges = [(s + 1, d + 1) for s, d in edges]
    rounds = [[np.eye(4)] + list(poses) for poses in rounds]
    got = {}
    for flags in (0, FLAG_NO_OBB):
        eng = Engine(flags=flags)
        eng.set_frames(pts, None); eng.set_graph(edges)
        got[flags] = []
        for poses in rounds:
            eng.set_poses(poses); eng.correspond(0.05)
            got[flags].append([eng.get_nn(e) for e in range(len(edges))])
        eng.close()
    for r, poses in enumerate(rounds):
        ref = oracle_correspond(O, pts, poses, edges, kind="brute", fixed0=False)
        for e, (s, d) in enumerate(edges):
            i0, d0 = got[0][r][e]
            i1, d1 = got[FLAG_NO_OBB][r][e]
            ni, nd = _numpy_nn(O, pts[s], pts[d], poses[s], poses[d])
            for name, (ii, dd) in (("per-lane search", (i1, d1)), ("oracle", (ref[e]["nn_idx"], ref[e]["nn_d2"])), ("numpy", (ni, nd))):
                assert np.array_equal(dd.view(np.uint64), d0.view(np.uint64)), (f"round {r} edge {e}: d2 differs from the {name}")
                assert np.array_equal(ii, i0), (f"round {r} edge {e}: {int((ii != i0).sum())} indices differ from the {name}")


def _sheet(rng, n, tilt=25.0):
    uv = rng.uniform(-0.1, 0.1, size=(n, 2))
    p = np.c_[uv, 0.002 * np.sin(40 * uv[:, 0])]
    return _f32(p @ _rot(rng, tilt).T)


def case_unrelated_clouds(O, n=6000):
    rng = np.random.default_rng(101)
    a = _f32(rng.normal(size=(n, 3)) * 0.05)
    b = _f32(rng.uniform(-0.3, 0.2, size=(n + 77, 3)) ** 3)
    c = _sheet(rng, n // 2)
    edges = [(0, 1), (1, 0), (2, 0), (0, 2)]
    I = [np.eye(4)] * 3
    moved = [_pose(rng, 20, [0.03, -0.02, 0.01]), np.eye(4), _pose(rng, -35, [0.0, 0.05, 0.0])]
    _check(O, [a, b, c], edges, [I, moved])


def case_volume_against_sheet(O, n=6000):
    rng = np.random.default_rng(102)
    vol = _f32(rng.uniform(-0.1, 0.1, size=(n, 3)))
    sheet = _sheet(rng, n)
    edges = [(0, 1), (1, 0)]
    _check(O, [vol, sheet], edges, [[np.eye(4)] * 2, [_pose(rng, 5, [0.01, 0, 0.02]), np.eye(4)]])


def case_pose_offset_of_many_diameters(O, n=5000):
    rng = np.random.default_rng(103)
    a = _f32(rng.normal(size=(n, 3)) * 0.02)      # diameter ~ 0.1
    b = _f32(a[rng.permutation(n)][: n - 13] + rng.normal(size=(n - 13, 3)) * 0.001)
    edges = [(0, 1), (1, 0)]
    far = [_pose(rng, 30, [7.0, -3.0, 5.0]), np.eye(4)]
    farther = [_pose(rng, 60, [-40.0, 25.0, 10.0]), _pose(rng, 10, [0.5, 0, 0])]
    _check(O, [a, b], edges, [far, farther])


def case_ties_and_duplicates(O, n=8):
    g = np.stack(np.meshgrid(np.arange(n), np.arange(n), np.arange(max(2, n // 2))), -1).reshape(-1, 3) / 64.0
    dup = np.repeat(g, 2, axis=0)[::-1].copy()        # every point twice, in reverse order: ties resolve to the lower index
    half = g + 0.5 / 64.0                             # every query equidistant from 8 grid points
    edges = [(1, 0), (2, 0), (0, 1)]
    shift = np.eye(4); shift[:3, 3] = [1 / 128.0, 0.0, 0.0]
    _check(O, [dup, half, g.copy()], edges, [[np.eye(4)] * 3, [np.eye(4), shift, np.eye(4)]])


def case_partial_warps(O, sizes=(1, 2, 5, 7, 8, 9, 16, 31, 32, 33, 40)):
    rng = np.random.default_rng(104)
    pts = [_f32(rng.normal(size=(k, 3)) * 0.01) for k in sizes]
    m = len(pts)
    edges = [(i, (i + 1) % m) for i in range(m)] + [(i, (i + 3) % m) for i in range(m)]
    moved = [_pose(rng, 3, rng.normal(size=3) * 0.01) for _ in range(m)]
    _check(O, pts, edges, [[np.eye(4)] * m, moved])


def case_partial_tiles(O, ks=(1, 2)):
    rng = np.random.default_rng(105)
    pts = [_f32(rng.normal(size=(1500, 3)) * 0.05)]
    for k in ks:
        for dn in (-1, 1):
            pts.append(_f32(rng.normal(size=(256 * k + dn, 3)) * 0.05))
    m = len(pts)
    edges = [(i, 0) for i in range(1, m)] + [(0, 1), (1, m - 1)]
    moved = [np.eye(4)] + [_pose(rng, 4, rng.normal(size=3) * 0.01) for _ in range(m - 1)]
    _check(O, pts, edges, [[np.eye(4)] * m, moved])


def case_georeferenced_fp64(O, n=4000):
    rng = np.random.default_rng(106)
    off = np.array([4.2e5, 1.3e6, 231.5])
    a = _sheet(rng, n) * 100.0 + rng.normal(size=(n, 3)) * 1e-3 + off   # not fp32-representable: fp64 records
    b = _sheet(rng, n + 5, tilt=-10.0) * 100.0 + rng.normal(size=(n + 5, 3)) * 1e-3 + off
    edges = [(0, 1), (1, 0)]
    P = np.eye(4); P[:3, 3] = [0.02, -0.01, 0.005]
    _check(O, [a, b], edges, [[np.eye(4)] * 2, [P, np.eye(4)]])


CASES = [case_unrelated_clouds, case_volume_against_sheet, case_pose_offset_of_many_diameters, case_ties_and_duplicates,
         case_partial_warps, case_partial_tiles, case_georeferenced_fp64]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.__name__[5:])
def test_far_rounds_match_per_lane_oracle_and_numpy(oracle, case):
    case(oracle)


def test_far_rounds_partial_tiles_of_many_sizes(oracle):
    case_partial_tiles(oracle, ks=(1, 3, 8))
