"""The three solves one after another on one engine: optimize, optimize_components, optimize_g2o, optimize after set_poses with
another fixed set, optimize_components.  They share the uploaded normal-equation layout, its states and its cache, so each call
must end exactly as the same call in a fresh engine that makes only that call from the same poses, fixed flags and
correspondences: poses, summary (and g2o's chi2 per call) bit for bit.

The graph has two components, one of them with a free frame whose only edge has no inlier (a column for the LM solves, none for
g2o); the wide case adds a 48-view component whose factor does not fit in shared memory."""
import numpy as np
import pytest

import test_gpu_components as T
import test_gpu_lm_graphs as G
from mv_lm_icp_b200 import COST_P2P, COST_P2PLANE, PARAM_SE3, Engine, synth
from mv_lm_icp_b200.api import default_g2o_options

pytestmark = pytest.mark.gpu


def cache_comps(O, n_points=1000, mode="f32", wide=False):
    kw = dict(n_points=n_points, mode=mode)
    comps = [T.Comp(O, 3, synth.ring_edges(3, 2), cfg=31, **kw),
             T.Comp(O, 4, [(1, 0), (2, 1), (1, 2), (2, 0), (3, 0)], empty=(4,), cfg=32, **kw)]
    if wide:
        assert G.skyline_bytes(48, G.wide_graph(48), (0,))[0] > G.SMEM_LIMIT
        comps.append(T.Comp(O, 48, G.wide_graph(48), cfg=33, n_points=min(n_points, 600), mode=mode))
    return comps


def _engine(b, mode, poses, fixed):
    """The batch's frames and graph, the given poses and fixed flags, and every edge's correspondences."""
    eng = Engine()
    eng.set_frames(b.pts, None if mode == "f32_no_normals" else b.nor)
    if mode == "f32_recomputed_normals":
        eng.recompute_normals(10)
    eng.set_graph(b.edges)
    eng.set_poses(poses, fixed)
    for e, (k, r) in enumerate(b.emap):
        c = b.comps[k]
        eng.set_edge(e, c.corr[r][0], c.corr[r][1], c.w[r])
    return eng


def _call(eng, kind, cost, lm_opts, g2o_opts):
    if kind == "optimize":
        return eng.optimize(PARAM_SE3, cost, True, options=lm_opts)
    if kind == "components":
        return eng.optimize_components(PARAM_SE3, cost, True, options=lm_opts)
    s, chi = eng.optimize_g2o(cost, options=g2o_opts)
    return s, T._bits(chi).tolist()


def check_sequence(O, comps, mode="f32", max_iter=None, g2o_calls=3):
    b = T.Batch(comps)
    cost = COST_P2P if mode == "f32_no_normals" else COST_P2PLANE
    lm_opts, _ = G._options(max_iter)
    g2o_opts = default_g2o_options(); g2o_opts.max_calls = g2o_calls
    lowest = [b.gid[k][0] for k in range(len(comps))]
    refix = [0] * b.M                     # another fixed set: frame 1 of every component instead of its lowest
    for k in range(len(comps)):
        refix[b.gid[k][1]] = 1
    calls = [("optimize", None), ("components", None), ("g2o", None), ("optimize", refix), ("components", None)]
    fixed = list(b.fx)
    eng = _engine(b, mode, b.poses, fixed)
    for i, (kind, new_fixed) in enumerate(calls):
        if new_fixed is not None:
            eng.set_poses(eng.get_poses(), new_fixed)
            fixed = list(new_fixed)
        poses = eng.get_poses()
        got = _call(eng, kind, cost, lm_opts, g2o_opts)
        P = eng.get_poses()
        fresh = _engine(b, mode, poses, fixed)
        want = _call(fresh, kind, cost, lm_opts, g2o_opts)
        Pf = fresh.get_poses()
        fresh.close()
        what = (i, kind, mode, len(comps))
        assert got == want, (what, got, want)
        assert np.array_equal(T._bits(P), T._bits(Pf)), what
        assert not np.array_equal(T._bits(P), T._bits(poses)), what     # the call did move something
        for f in ([0] if kind != "components" else lowest):            # what the call fixed
            fixed[f] = 1
    eng.close()


@pytest.mark.parametrize("mode", G.MODES)
def test_sequence_matches_fresh_engines(oracle, mode):
    check_sequence(oracle, cache_comps(oracle, mode=mode), mode)


def test_sequence_with_factor_in_global_memory(oracle):
    check_sequence(oracle, cache_comps(oracle, wide=True))
