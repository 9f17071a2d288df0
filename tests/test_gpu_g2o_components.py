"""One g2o problem per connected component (Engine.optimize_g2o_components / mvicp_optimize_g2o_components).

Contract: every component ends exactly as Engine.optimize_g2o ends in a fresh engine that holds only that component (its frames
in ascending order, its edges in graph order, the same fixed flags, options and correspondences) -- poses, every summary field,
chi2 per call and the trial trace (up to the rows the batch records) bit for bit -- as long as the settings the batch shares are
the same there: the streaming tile length and the storage mode.  Those preconditions are asserted, and each component is also
held to tests/g2o_model.py under the contract of tests/test_gpu_g2o.py (check_against_model).  On a connected graph the call
equals Engine.optimize_g2o."""
import numpy as np
import pytest

import test_gpu_lm_graphs as G
from helpers import scene
from mv_lm_icp_b200 import COST_MIXED, COST_P2P, COST_P2PLANE, PARAM_SE3, Engine, MvicpError, default_g2o_options, synth
from test_gpu_components import Batch, Comp, _bits
from test_gpu_g2o import check_against_model
from test_gpu_g2o_graphs import G2O_TOPOLOGIES, fixed_flags, g2o_topology, graph_corr, short_options, upload

pytestmark = pytest.mark.gpu
ERR_INVALID, ERR_STATE = 1, 4                                     # MVICP_ERR_*
END_NO_IMPROVEMENT, END_MAX_CALLS, END_NO_VERTICES = 0, 1, 2      # MVICP_G2O_END_*
NO_VERTICES = {"calls": 0, "iterations": 0, "trials": 0, "accepted": 0, "evaluations": 0, "ended": END_NO_VERTICES,
               "last_call_end": 0, "chi2_initial": 0.0, "chi2_final": 0.0}


def trace_cap(n_problems):
    """Trial rows the batch records per problem (mvicp.cu: max(G2O_TRACE_MIN, G2O_TRACE_CAP / P))."""
    return max(1024, 65536 // n_problems)


class Raw:
    """A component given by its arrays, with the attributes of test_gpu_components.Comp that Batch and the checks read."""

    def __init__(self, pts, nor, poses, edges, corr, fixed=()):
        self.pts, self.nor, self.poses, self.edges, self.corr = pts, nor, poses, list(edges), list(corr)
        self.n = len(pts)
        self.fx = G._fixed_list(self.n, fixed)
        self.fx[0] = 1
        self.free = not all(self.fx)
        self.w = [np.float32(1)] * len(edges)

    def active_slots(self):
        return sum(len(self.pts[s]) for s, _ in self.edges if not self.fx[s])


def _load(eng, pts, nor, poses, fx, edges, corr_of_edge, mode):
    """Frames, graph, poses, fixed flags and the correspondences of EVERY edge (g2o uses the edges of fixed src frames too);
    returns the normals the solve reads."""
    eng.set_frames(pts, None if mode == "f32_no_normals" else nor)
    out = nor
    if mode == "f32_recomputed_normals":
        out, _ = eng.recompute_normals(10)
    if mode == "f32_no_normals":
        out = [None] * len(pts)
    eng.set_graph(edges)
    eng.set_poses(poses, fx)
    for e in range(len(edges)):
        first, second, w = corr_of_edge(e)
        eng.set_edge(e, first, second, w)
    return out


def _batch_corr(b):
    def corr(e):
        k, r = b.emap[e]
        return b.comps[k].corr[r][0], b.comps[k].corr[r][1], b.comps[k].w[r]
    return corr


def solve_batch(b, cost, opts, mode="f32"):
    """optimize_g2o_components on the batch: (poses, [(summary, chi2 per call, trace)] per component, normals used)."""
    eng = Engine()
    nor = _load(eng, b.pts, b.nor, b.poses, b.fx, b.edges, _batch_corr(b), mode)
    n, comp_of = eng.components()
    assert n == len(b.comps)
    for k in range(n):
        assert all(comp_of[g] == k for g in b.gid[k])
    res = eng.optimize_g2o_components(cost, opts)
    out = [(s, chis, eng.g2o_trace(component=k)) for k, (s, chis) in enumerate(res)]
    P = eng.get_poses()
    eng.close()
    return P, out, nor


def fresh_engine(c, mode="f32"):
    eng = Engine()
    nor = _load(eng, c.pts, c.nor, c.poses, c.fx, c.edges, lambda e: (c.corr[e][0], c.corr[e][1], c.w[e]), mode)
    return eng, nor


def check_batch(comps, cost=COST_P2PLANE, opts=None, mode="f32", model=True):
    """The batch against a fresh engine per component, bit for bit, and (model) every component against tests/g2o_model.py.
    Returns [(summary, chi2 per call, trace)] per component."""
    opts = short_options() if opts is None else opts
    b = Batch(comps)
    tl = G.tile_len(b.active_slots())
    P, out, nor = solve_batch(b, cost, opts, mode)
    cap = trace_cap(max(1, sum(1 for s, _, _ in out if s["ended"] != END_NO_VERTICES)))
    for k, c in enumerate(comps):
        Pk, (sk, chk, trk) = P[b.gid[k]], out[k]
        what = (k, c.n, cost, mode, sk)
        assert len(trk) == sk["trials"], what
        if sk["ended"] == END_NO_VERTICES:
            assert sk == NO_VERTICES and chk.tolist() == [0.0], what
            assert np.array_equal(_bits(Pk), _bits(c.poses)), what
        if not c.edges:                   # an isolated frame: a context without edges cannot solve
            continue
        # preconditions of the bit-for-bit contract: the settings the batch shares are this component's own
        assert G.tile_len(c.active_slots()) == tl, (what, c.active_slots(), b.active_slots())
        eng, nk = fresh_engine(c, mode)
        eng.set_poses(c.poses, c.fx)
        sf, chf = eng.optimize_g2o(cost, opts)
        Pf, trf = eng.get_poses(), eng.g2o_trace()
        assert sk == sf, (what, sf)
        assert np.array_equal(_bits(chk), _bits(chf)), what
        assert len(trk) == len(trf) and np.array_equal(_bits(trk[:cap]), _bits(trf[:cap])), what
        assert np.array_equal(_bits(Pk), _bits(Pf)), what
        if model and sk["ended"] != END_NO_VERTICES:
            check_against_model(eng, c.pts, nk, c.poses, c.edges, np.array(c.fx, np.uint8), cost, opts)
        eng.close()
    return out


# ---- 1. connected graphs: the call is mvicp_optimize_g2o -----------------------------------------------------------------
CONNECTED = [t for t in G2O_TOPOLOGIES if t != "two_components"]


def check_connected(O, name, costs=(COST_P2P, COST_P2PLANE), paths=("rigid", "nonrigid"), n_points=1500, opts=None):
    M, edges, fixed, empty, src0 = g2o_topology(name)
    sc = scene(M, n_points, 43)
    views = G.HUB_RING if name == "hub_last" else list(range(M))
    order = [views.index(f) for f in range(M)]
    pts, nor = [sc["pts"][v] for v in order], [sc["nor"][v] for v in order]
    poses0 = sc["poses_init"][order].copy()
    corr = graph_corr(O, pts, poses0, edges, empty, src0)
    fx = fixed_flags(M, fixed)
    engs = [Engine(), Engine()]
    for eng in engs:
        eng.set_frames(pts, nor); eng.set_graph(edges); upload(eng, corr)
    assert engs[1].components()[0] == 1
    for path in paths:
        poses = poses0.copy()
        if path == "nonrigid":
            poses[1] = G._nonrigid(poses[1])
        for cost in costs:
            out = []
            for i, eng in enumerate(engs):
                eng.set_poses(poses, fx)
                if i == 0:
                    s, chis = eng.optimize_g2o(cost, opts)
                    trace = eng.g2o_trace()
                else:
                    (s, chis), = eng.optimize_g2o_components(cost, opts)
                    trace = eng.g2o_trace(component=0)
                out.append((eng.get_poses(), s, chis, trace))
            what = (name, path, cost)
            assert out[0][1] == out[1][1], (what, out[0][1], out[1][1])
            for j in (0, 2, 3):
                assert np.array_equal(_bits(out[0][j]), _bits(out[1][j])), (what, j)
    for eng in engs:
        eng.close()


@pytest.mark.parametrize("name", CONNECTED)
def test_connected_graph_equals_optimize_g2o(oracle, name):
    check_connected(oracle, name)


# ---- 2. mixed batches --------------------------------------------------------------------------------------------------
def mixed_comps(O, n_points=1200, mode="f32", wide=True):
    """Two-view pairs, a ring with chords, a ring with a user-fixed frame that is not its lowest (whose out-edges carry
    matches: active in g2o), an all-fixed ring and an isolated frame (no vertex), a component with a free frame without
    inliers (not a vertex), a non-rigid ring and (wide) a 48-view component whose factor needs global memory."""
    kw = dict(n_points=n_points, mode=mode)
    comps = [
        Comp(O, 2, [(1, 0), (0, 1)], cfg=11, **kw),
        Comp(O, 6, synth.ring_edges(6, 2) + [(1, 4), (4, 1)], cfg=12, **kw),
        Comp(O, 2, [(0, 1), (1, 0)], cfg=13, **kw),
        Comp(O, 5, synth.ring_edges(5, 2), fixed=(2,), cfg=14, **kw),
        Comp(O, 3, synth.ring_edges(3, 1), fixed=(0, 1, 2), cfg=15, **kw),
        Comp(O, 1, [], cfg=16, **kw),
        Comp(O, 4, [(1, 0), (2, 1), (1, 2), (2, 0), (3, 0)], empty=(4,), cfg=17, **kw),
        Comp(O, 3, synth.ring_edges(3, 2), cfg=19, nonrigid=True, **kw),
    ]
    assert len(comps[3].corr[synth.ring_edges(5, 2).index((2, 3))][0]) > 0     # an edge out of the fixed frame 2 with matches
    if wide:
        comps.append(Comp(O, 48, G.wide_graph(48), cfg=18, n_points=600, mode=mode))
    return comps


@pytest.mark.parametrize("cost", [COST_P2P, COST_P2PLANE])
def test_batch_matches_fresh_engines_and_model(oracle, cost):
    comps = mixed_comps(oracle)
    assert G.skyline_bytes(48, G.wide_graph(48), (0,))[0] > G.SMEM_LIMIT      # every frame of it is a vertex: LM's profile
    out = check_batch(comps, cost)
    ended = [s["ended"] for s, _, _ in out]
    assert ended[4] == ended[5] == END_NO_VERTICES and ended.count(END_NO_VERTICES) == 2, ended
    # one call of short_options: every component with a vertex ends on MAX_CALLS, each with its own chi2
    assert all(s["ended"] == END_MAX_CALLS for k, (s, _, _) in enumerate(out) if k not in (4, 5)), ended
    assert len({s["chi2_final"] for s, _, _ in out}) == len(out) - 1


# ---- 3. mixed outcomes ---------------------------------------------------------------------------------------------------
def failing_pair(seed=17, n=300):
    """Every match's src point sits at the origin (test_gpu_g2o_graphs.test_failed_factorisation_is_a_rejected_trial): with
    tau = 0 every trial's factorisation fails, each call ends on Terminate and the outer loop on no improvement."""
    rng = np.random.default_rng(seed)
    dst = (rng.normal(size=(n, 3)) * 0.1).astype(np.float32).astype(np.float64)
    src = (rng.normal(size=(n, 3)) * 0.1).astype(np.float32).astype(np.float64)
    src[:40] = 0.0
    nor = [G._unit(rng, n).astype(np.float32).astype(np.float64) for _ in range(2)]
    poses = np.stack([np.eye(4), G._rigid(rng, 0.05, 0.02)])
    corr = [(np.arange(40, dtype=np.int32), rng.choice(n, 40, replace=False).astype(np.int32))]
    return Raw([dst, src], nor, poses, [(1, 0)], corr)


@pytest.mark.parametrize("ortho_after", [1000, 2])
def test_mixed_outcomes_in_one_batch(oracle, ortho_after, n_points=1200):
    """A failed factorisation next to converging components; a component that ends on MAX_CALLS next to one that ends on
    NO_IMPROVEMENT.  The healthy components' bits do not depend on the failing one being in the batch."""
    o = default_g2o_options(); o.tau = 0.0; o.max_calls = 8; o.iterations_per_call = 1; o.orthonormalize_after = ortho_after
    healthy = [Comp(oracle, 2, [(1, 0)], cfg=21, n_points=n_points), Comp(oracle, 4, synth.ring_edges(4, 2), cfg=22, n_points=n_points)]
    out = check_batch([failing_pair()] + healthy, COST_P2P, o, model=False)
    s0, _, tr0 = out[0]
    assert s0["ended"] == END_NO_IMPROVEMENT and s0["accepted"] == 0 and np.all(tr0[:, 2] == np.inf), s0
    assert s0["trials"] == s0["calls"] * o.max_trials
    assert any(s["ended"] == END_MAX_CALLS for s, _, _ in out[1:]), [s for s, _, _ in out]
    alone = check_batch(healthy, COST_P2P, o, model=False)
    for (a, ca, ta), (b, cb, tb) in zip(out[1:], alone):
        assert a == b and np.array_equal(_bits(ca), _bits(cb)) and np.array_equal(_bits(ta), _bits(tb))


# ---- 4. storage modes ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", G.MODES)
def test_storage_modes(oracle, mode):
    comps = [Comp(oracle, 2, [(1, 0), (0, 1)], cfg=31, n_points=1000, mode=mode),
             Comp(oracle, 5, synth.ring_edges(5, 2), fixed=(2,), cfg=32, n_points=1000, mode=mode),
             Comp(oracle, 4, [(1, 0), (2, 1), (1, 2), (2, 0), (3, 0)], empty=(4,), cfg=33, n_points=1000, mode=mode)]
    check_batch(comps, COST_P2P, mode=mode)
    if mode == "f32_no_normals":
        b = Batch(comps)
        eng = Engine(); _load(eng, b.pts, b.nor, b.poses, b.fx, b.edges, _batch_corr(b), mode)
        with pytest.raises(MvicpError) as ei:
            eng.optimize_g2o_components(COST_P2PLANE)
        assert ei.value.code == ERR_INVALID
        eng.close()
    else:
        check_batch(comps, COST_P2PLANE, mode=mode)


# ---- 5. every solve on one engine ----------------------------------------------------------------------------------------
def check_one_engine(O, n_points=1200):
    """optimize, optimize_components, optimize_g2o, optimize_g2o_components, optimize on one engine (one layout cache), each
    from the same start, equal a fresh engine that makes only that call.  The lowest frame of every component is user-fixed,
    so that the joint solves are well posed."""
    comps = [Comp(O, 2, [(1, 0)], cfg=41, n_points=n_points), Comp(O, 4, synth.ring_edges(4, 2) + [(3, 1)], cfg=42, n_points=n_points)]
    b = Batch(comps)
    fx = list(b.fx)
    for k in range(len(comps)):
        fx[b.gid[k][0]] = 1

    def solve(eng, kind):
        eng.set_poses(b.poses, fx)
        if kind == "lm":
            s = eng.optimize(PARAM_SE3, COST_P2PLANE, True)
        elif kind == "lm_comp":
            s = eng.optimize_components(PARAM_SE3, COST_P2PLANE, True)
        elif kind == "g2o":
            sg, chis = eng.optimize_g2o(COST_P2PLANE)
            s = (sg, chis.tolist(), eng.g2o_trace().tolist())
        else:
            s = [(sg, chis.tolist(), eng.g2o_trace(component=k).tolist())
                 for k, (sg, chis) in enumerate(eng.optimize_g2o_components(COST_P2PLANE))]
        return eng.get_poses(), repr(s)

    def fresh():
        eng = Engine(); _load(eng, b.pts, b.nor, b.poses, fx, b.edges, _batch_corr(b), "f32")
        return eng
    kinds = ["lm", "lm_comp", "g2o", "g2o_comp", "lm"]
    eng = fresh()
    got = [solve(eng, k) for k in kinds]
    eng.close()
    for k, g in zip(kinds, got):
        e2 = fresh(); want = solve(e2, k); e2.close()
        assert np.array_equal(_bits(g[0]), _bits(want[0])), k
        assert g[1] == want[1], (k, g[1], want[1])


def test_every_solve_on_one_engine(oracle):
    check_one_engine(oracle)


# ---- 6. ICP rounds: correspond + optimize_g2o_components -----------------------------------------------------------------
def check_icp_rounds(n_pairs=8, n_points=3000, rounds=20, thresh=0.05):
    pairs = [scene(2, n_points, 100 + i) for i in range(n_pairs)]
    pts = [p["pts"][0] for p in pairs] + [p["pts"][1] for p in pairs]
    nor = [p["nor"][0] for p in pairs] + [p["nor"][1] for p in pairs]
    poses = np.concatenate([np.stack([p["poses_init"][0] for p in pairs]), np.stack([p["poses_init"][1] for p in pairs])])
    g_edges = [(n_pairs + i, i) for i in range(n_pairs)] + [(i, n_pairs + i) for i in range(n_pairs)]
    eng = Engine(); eng.set_frames(pts, nor); eng.set_graph(g_edges); eng.set_poses(poses, [1] * n_pairs + [0] * n_pairs)
    fresh = []
    for p in pairs:
        f = Engine(); f.set_frames(p["pts"], p["nor"]); f.set_graph([(1, 0), (0, 1)]); f.set_poses(p["poses_init"]); fresh.append(f)
    assert G.tile_len(n_points * n_pairs) == G.tile_len(n_points)
    for rnd in range(rounds):
        eng.correspond(thresh)
        res = eng.optimize_g2o_components(COST_P2PLANE)
        P = eng.get_poses()
        for i, f in enumerate(fresh):
            f.correspond(thresh)
            s, chis = f.optimize_g2o(COST_P2PLANE)
            assert res[i][0] == s and np.array_equal(_bits(res[i][1]), _bits(chis)), (rnd, i, res[i][0], s)
            assert np.array_equal(_bits(eng.g2o_trace(component=i)), _bits(f.g2o_trace())), (rnd, i)
            assert np.array_equal(_bits(P[[i, n_pairs + i]]), _bits(f.get_poses())), (rnd, i)
    for f in [eng] + fresh:
        f.close()


def test_icp_rounds_equal_one_engine_per_pair():
    check_icp_rounds()


# ---- 7. API --------------------------------------------------------------------------------------------------------------
def check_api(n_points=500):
    sc = scene(7, n_points, 31)
    eng = Engine()
    eng.set_frames(sc["pts"], None)
    with pytest.raises(MvicpError) as ei:
        eng.optimize_g2o_components(COST_P2P)                   # no graph yet
    assert ei.value.code == ERR_STATE
    edges = [(3, 1), (5, 3), (2, 6), (1, 3)]
    eng.set_graph(edges)
    assert eng.components()[0] == 4 and list(eng.components()[1]) == [0, 1, 2, 1, 3, 1, 2]
    eng.set_poses(sc["poses_init"], [0] * 7)
    eng.correspond(0.05)
    assert eng.stats()["queries"] == 4 * n_points
    bad = default_g2o_options(); bad.max_calls = 0
    for cost, o in ((COST_MIXED, None), (COST_P2PLANE, None), (COST_P2P, bad)):   # bad cost, no normals, bad options
        with pytest.raises(MvicpError) as ei:
            eng.optimize_g2o_components(cost, o)
        assert ei.value.code == ERR_INVALID
    eng.correspond(0.05)                                        # rejected calls fixed no frame: every edge is still searched
    assert eng.stats()["queries"] == 4 * n_points
    o = default_g2o_options(); o.max_calls = 3
    res = eng.optimize_g2o_components(COST_P2P, o)
    assert len(res) == 4
    assert res[0][0] == NO_VERTICES and res[3][0] == NO_VERTICES and res[0][1].tolist() == [0.0]
    for k in (1, 2):
        s, chis = res[k]
        assert s["ended"] != END_NO_VERTICES and s["calls"] <= 3 and len(chis) == s["calls"] + 1 and chis[0] == s["chi2_initial"]
        tr = eng.g2o_trace(component=k)
        assert tr.shape == (s["trials"], 5) and s["trials"] > 0
    assert len(eng.g2o_trace(component=0)) == 0
    with pytest.raises(MvicpError) as ei:
        eng.g2o_trace()                                         # the last g2o solve ran per component
    assert ei.value.code == ERR_STATE
    for k in (-1, 4):
        with pytest.raises(MvicpError) as ei:
            eng.g2o_trace(component=k)
        assert ei.value.code == ERR_INVALID
    P = eng.get_poses()
    for f in (0, 4):                                            # components without a vertex keep their poses
        assert np.array_equal(_bits(P[f]), _bits(sc["poses_init"][f])), f
    eng.correspond(0.05)                                        # the lowest frames 1 and 2 are fixed now
    assert eng.stats()["queries"] == 2 * n_points
    s, _ = eng.optimize_g2o(COST_P2P, o)                        # after the joint solve both trace calls work and agree
    assert np.array_equal(eng.g2o_trace(), eng.g2o_trace(component=0)) and len(eng.g2o_trace()) == s["trials"]
    with pytest.raises(MvicpError) as ei:
        eng.g2o_trace(component=1)
    assert ei.value.code == ERR_INVALID
    eng.close()


def test_api():
    check_api()
