"""Checks of the g2o restatement (tests/g2o_model.py) that do not depend on the engine: the analytic Jacobians against central
differences of the error through the oplus update, chi2 against a per-correspondence evaluation with makeRot0 / prec0 written
out, the increment and orthonormalisation rules, and a committed LM trace (tests/golden/g2o_trace.npz, make_golden.py)."""
import os

import numpy as np
import pytest

import g2o_model as G

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _pose(rng, nonrigid):
    w = rng.normal(size=3) * 0.7
    th = np.linalg.norm(w); k = w / th
    K = G.skew(k)[0]
    T = np.eye(4); T[:3, :3] = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K; T[:3, 3] = rng.normal(size=3) * 0.3
    if nonrigid:
        T[:3, :3] = T[:3, :3] @ np.diag([1.0, 0.9957, 0.9957]) @ (np.eye(3) + 0.01 * rng.normal(size=(3, 3)))
    return T


@pytest.mark.parametrize("nonrigid", [False, True])
def test_jacobians_are_central_differences_through_oplus(nonrigid):
    """J_src is the derivative of e through T1 <- T1 inc at any pose; J_dst's rotation columns are, too.  J_dst's translation
    block is g2o's -I: the true derivative is -F0^T F0, equal to -I only for a rigid F0 -- both are asserted."""
    rng = np.random.default_rng(5 + nonrigid)
    T0, T1 = _pose(rng, nonrigid), _pose(rng, nonrigid)
    p0 = rng.normal(size=(7, 3)); p1 = rng.normal(size=(7, 3))
    Jd, Js = G.jacobians(T0, T1, p1)
    h = 1e-6
    for k in range(6):
        d = np.zeros(6); d[k] = h
        for which, J in (("src", Js), ("dst", Jd)):
            Tp = G.oplus(T1 if which == "src" else T0, d, 0, 1000)[0]
            Tm = G.oplus(T1 if which == "src" else T0, -d, 0, 1000)[0]
            ep = G.error(T0, Tp, p0, p1) if which == "src" else G.error(Tp, T1, p0, p1)
            em = G.error(T0, Tm, p0, p1) if which == "src" else G.error(Tm, T1, p0, p1)
            fd = (ep - em) / (2 * h)
            want = J[:, :, k]
            if which == "dst" and k < 3:
                F0 = T0[:3, :3]
                want_true = np.broadcast_to(-(F0.T @ F0)[:, k], fd.shape)
                assert np.max(np.abs(fd - want_true)) <= 1e-7 * max(1.0, np.max(np.abs(want_true)))
                if nonrigid:
                    assert np.max(np.abs(want - want_true)) > 1e-4   # g2o keeps -I
                    continue
            assert np.max(np.abs(fd - want)) <= 1e-7 * max(1.0, np.max(np.abs(want))), (which, k)


def test_chi2_matches_a_per_correspondence_evaluation():
    rng = np.random.default_rng(11)
    pts = [rng.normal(size=(40, 3)) for _ in range(3)]
    nor = [rng.normal(size=(40, 3)) * 1.3 for _ in range(3)]   # not unit: prec0 differs from eps I + (1 - eps) n n^T
    poses = [np.eye(4), _pose(rng, True), _pose(rng, False)]
    edges = [(1, 0), (2, 1), (0, 2)]
    corr = [(rng.permutation(40)[:25], rng.integers(0, 40, 25)) for _ in edges]
    for plane in (False, True):
        prob = G.Problem(pts, nor, edges, corr, [True, False, False], plane, eps=0.01)
        want = 0.0
        for (s, d), (f, sec) in zip(edges, corr):
            F0, t0, F1, t1 = poses[d][:3, :3], poses[d][:3, 3], poses[s][:3, :3], poses[s][:3, 3]
            for a, b in zip(f, sec):
                e = F0.T @ (F1 @ pts[s][a] + t1) - F0.T @ t0 - pts[d][b]
                if plane:
                    n = nor[d][b]
                    y = np.array([0.0, 1.0, 0.0]) - n[1] * n; y = y / np.linalg.norm(y)
                    R0 = np.array([np.cross(n, y), y, n])
                    Om = R0.T @ np.diag([0.01, 0.01, 1.0]) @ R0
                    assert not np.allclose(Om, 0.01 * np.eye(3) + 0.99 * np.outer(n, n))
                else:
                    Om = np.eye(3)
                want += e @ Om @ e
        assert prob.chi2(poses) == pytest.approx(want, rel=1e-13)


def test_increment_and_orthonormalisation():
    T = np.eye(4)
    R = G.increment(np.array([0, 0, 0, 0.8, 0.7, 0.1]))   # |q|^2 > 1: identity rotation
    assert np.array_equal(R[:3, :3], np.eye(3))
    q = np.array([0.1, -0.2, 0.05]); R = G.increment(np.r_[0.0, 0.0, 0.0, q])[:3, :3]
    assert np.allclose(R @ R.T, np.eye(3), atol=1e-15) and np.isclose(np.linalg.det(R), 1.0)
    F = np.diag([1.0, 0.99, 1.01]); T[:3, :3] = F
    out, c = G.oplus(T, np.zeros(6), 3, 3)   # the 4th update passes orthonormalize_after = 3
    assert c == 0 and np.allclose(out[:3, :3], F - 0.5 * F @ (F.T @ F - np.eye(3)))
    out, c = G.oplus(T, np.zeros(6), 2, 3)
    assert c == 3 and np.array_equal(out[:3, :3], F)


def golden_problem():
    """The trace fixture's problem: three frames of a random cloud, point-to-plane.  Frame 1, a free dst frame, starts strongly
    non-rigid: g2o's -I translation block of J_dst is then not the derivative (-F0^T F0), trials overshoot and are rejected,
    so the kept trace exercises the rejection branch (lambda *= nu, nu *= 2) as well as acceptance."""
    rng = np.random.default_rng(2024)
    base = rng.normal(size=(300, 3)) * 0.1
    nor = rng.normal(size=(300, 3)); nor /= np.linalg.norm(nor, axis=1)[:, None]
    truth = [np.eye(4), _pose(rng, False), _pose(rng, False)]
    pts = [(base - T[:3, 3]) @ T[:3, :3] for T in truth]       # frame f sees base in its own coordinates
    nors = [nor @ T[:3, :3] for T in truth]
    start = [truth[0]] + [T @ G.oplus(np.eye(4), rng.normal(size=6) * 0.02, 0, 1000)[0] for T in truth[1:]]
    start[1][:3, :3] = start[1][:3, :3] @ np.diag([1.0, 0.8, 1.25])
    idx = np.arange(300)
    edges = [(1, 0), (2, 1), (2, 0)]
    return pts, nors, edges, [(idx, idx)] * 3, start


def test_committed_trace():
    pts, nor, edges, corr, start = golden_problem()
    prob = G.Problem(pts, nor, edges, corr, [True, False, False], True)
    P, summ, chis, trace = G.optimize(prob, start)
    g = np.load(os.path.join(GOLDEN, "g2o_trace.npz"))
    k = len(g["trace"])
    assert len(trace) >= k and k >= 10 and (g["trace"][:, 4] == 0).sum() >= 5   # rejected trials are part of the fixture
    np.testing.assert_allclose(trace[:k], g["trace"], rtol=1e-9, atol=1e-300)
    np.testing.assert_allclose(P, g["poses"], atol=1e-10)
    assert summ["calls"] == int(g["calls"])
