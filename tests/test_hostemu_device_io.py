"""The device twins of the C ABI (mvicp_*_device, mvicp_closest_points) on the host model of CUDA (tools/hostemu), where every
allocation stands for device memory: numpy buffers are passed where a caller on the GPU would pass device pointers.  Each twin
must return the same bytes as its host-memory counterpart; this checks their logic (argument checks, the set_edge range check
and last-occurrence rule, the compaction into a caller's buffer) in ascending and random thread order.  The GPU suite
(tests/test_gpu_device_io.py) checks the same on the hardware, with torch tensors."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools", "hostemu"))

INVALID, STATE = 1, 4


@pytest.fixture(scope="module", params=["ascending", "random"])
def emu(request, tmp_path_factory):
    import shutil
    import build_hostemu
    from mv_lm_icp_b200 import _lib
    so = build_hostemu.build()
    if request.param == "random":       # the order is read once when the library is loaded: load a private copy
        so2 = str(tmp_path_factory.mktemp("hostemu_io") / "libmvicp_hostemu_random.so")
        shutil.copy(so, so2); so = so2
        os.environ["HOSTEMU_ORDER"] = "random"
    lib = C.CDLL(so); lib.mvicp_last_error.restype = C.c_char_p
    os.environ.pop("HOSTEMU_ORDER", None)
    saved = _lib._lib
    _lib._lib = lib
    yield lib
    _lib._lib = saved


def _vp(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def _scene(n_views=3, n_points=400):
    from mv_lm_icp_b200 import synth
    return synth.make_scene(n_views, n_points, config_id=1)


def _set_frames_device(eng, pts, nor):
    M = len(pts)
    PP = (C.c_void_p * M)(*[p.ctypes.data for p in pts])
    NN = None if nor is None else (C.c_void_p * M)(*[n.ctypes.data for n in nor])
    n = np.ascontiguousarray([len(p) for p in pts], np.int64)
    rc = eng._l.mvicp_set_frames_device(eng._ctx, C.c_int32(M), PP, NN, n.ctypes.data_as(C.POINTER(C.c_int64)))
    assert rc == 0, eng._l.mvicp_last_error()
    eng.M = M; eng.n_pts = [len(p) for p in pts]


def _all_edges_device(eng):
    E = len(eng.edges)
    cap = sum(eng.n_pts[s] for s, _ in eng.edges)
    rec = np.full(cap, 0x5A, np.dtype([("first", np.int32), ("second", np.int32), ("dist", np.float64)]))
    off = np.full(E + 1, -7, np.int64); w = np.full(E, np.nan, np.float32)
    rc = eng._l.mvicp_get_all_edges_device(eng._ctx, _vp(rec), C.c_int64(cap), _vp(off), _vp(w))
    assert rc == 0, eng._l.mvicp_last_error()
    return rec[:off[E]], off, w


def _same_edges(a, b):
    ra, oa, wa = a; rb, ob, wb = b
    assert np.array_equal(oa, ob)
    assert ra.tobytes() == rb.tobytes()
    assert wa.view(np.uint32).tolist() == wb.view(np.uint32).tolist()


def _host_edges(eng):
    eng.pull_all_edges()
    off = eng.edge_offsets
    return eng._rec_buf[:off[-1]].copy(), off.copy(), np.array([w for _, w in eng.host_edges], np.float32)


@pytest.mark.parametrize("mode", ["fp32", "fp64", "p2p", "recomputed_normals"])
def test_set_frames_device_twin(emu, mode):
    """Two engines, one loaded through mvicp_set_frames, one through mvicp_set_frames_device (its input overwritten with NaN
    right after the call): identical poses and edge lists over three ICP rounds."""
    from mv_lm_icp_b200 import COST_P2P, COST_P2PLANE, Engine, synth
    sc = _scene()
    pts = [p.copy() for p in sc["pts"]]
    if mode == "fp64":
        rng = np.random.default_rng(3)
        pts = [p + rng.normal(0, 1e-7, p.shape) for p in pts]
    nor = None if mode in ("p2p", "recomputed_normals") else [n.copy() for n in sc["nor"]]
    edges = synth.ring_edges(3, 2)
    engs = []
    for dev in (False, True):
        eng = Engine()
        if dev:
            P = [p.copy() for p in pts]; N = None if nor is None else [n.copy() for n in nor]
            _set_frames_device(eng, P, N)
            for a in P + (N or []):
                a[:] = np.nan
        else:
            eng.set_frames(pts, nor)
        if mode == "recomputed_normals":
            eng.recompute_normals(10, fetch=False)
        eng.set_graph(edges); eng.set_poses(sc["poses_init"])
        engs.append(eng)
    cost = COST_P2P if mode == "p2p" else COST_P2PLANE
    for _ in range(3):
        sa, sb = (e.icp_round(0.05, cost=cost) for e in engs)
        assert sa == sb
        Pa, Pb = (e.get_poses() for e in engs)
        assert Pa.tobytes() == Pb.tobytes()
        _same_edges(_host_edges(engs[0]), _host_edges(engs[1]))
    for e in engs:
        e.close()


def test_get_all_edges_device_twin(emu):
    """mvicp_get_all_edges_device writes what mvicp_get_all_edges returns; NULL records; capacity one below the bound is
    refused before anything is written; before mvicp_correspond it is a state error."""
    from mv_lm_icp_b200 import Engine, synth
    sc = _scene()
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(synth.ring_edges(3, 2)); eng.set_poses(sc["poses_init"])
    E = len(eng.edges)
    off = np.zeros(E + 1, np.int64)
    assert eng._l.mvicp_get_all_edges_device(eng._ctx, None, C.c_int64(0), _vp(off), None) == STATE
    for cut in (0.05, 0.0004):
        eng.correspond(cut)
        _same_edges(_host_edges(eng), _all_edges_device(eng))
        off2 = np.zeros(E + 1, np.int64)
        assert eng._l.mvicp_get_all_edges_device(eng._ctx, None, C.c_int64(0), _vp(off2), None) == 0
        assert np.array_equal(off2, eng.edge_offsets)
    bound = sum(eng.n_pts[s] for s, _ in eng.edges if s != 0)
    rec = np.full(bound, 0x33, np.uint8).repeat(16); off3 = np.full(E + 1, 0x44, np.int64)
    assert eng._l.mvicp_get_all_edges_device(eng._ctx, _vp(rec), C.c_int64(bound - 1), _vp(off3), None) == INVALID
    assert np.all(rec == 0x33) and np.all(off3 == 0x44)
    assert eng._l.mvicp_get_all_edges_device(eng._ctx, _vp(rec), C.c_int64(bound), _vp(off3), None) == 0
    eng.close()


def test_closest_points_twins(emu):
    """mvicp_closest_points and its device twin equal mvicp_closest_point query by query: near and far queries, copies of cloud
    points, a duplicated point (lowest index), a 1e5 offset (fp64 storage), non-finite queries (-1, NaN), n = 0, a bad frame."""
    from mv_lm_icp_b200 import Engine
    sc = _scene()
    cloud = sc["pts"][1].copy()
    cloud[7] = cloud[300]                               # a duplicated point: the tie goes to index 7
    rng = np.random.default_rng(5)
    q = np.concatenate([cloud[rng.integers(len(cloud), size=40)] + rng.normal(0, 0.003, (40, 3)),
                        cloud[[0, 7, 300, len(cloud) - 1]],
                        rng.normal(0, 1e3, (6, 3)),
                        np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf]])])
    q0 = q
    for off in (0.0, 1e5):                              # fp32 storage / fp64 storage (the offset is not fp32-representable)
        pts = [sc["pts"][0], cloud + off]
        q = q0 + off
        eng = Engine(); eng.set_frames(pts, None)
        idx = np.full(len(q), -9, np.int64); d2 = np.zeros(len(q))
        assert eng._l.mvicp_closest_points_device(eng._ctx, 1, _vp(q), C.c_int64(len(q)), _vp(idx), _vp(d2)) == 0
        hi, hd = eng.closest_points(1, q)
        assert np.array_equal(hi, idx) and hd.tobytes() == d2.tobytes()
        for i, x in enumerate(q):
            if np.all(np.isfinite(x)):
                ri, rd = eng.closest_point(1, x)
                assert ri == idx[i] and np.float64(rd).tobytes() == d2[i].tobytes(), i
            else:
                assert idx[i] == -1 and np.isnan(d2[i])
        assert idx[41] == 7 and idx[42] == 7 and d2[41] == 0.0
        assert eng._l.mvicp_closest_points_device(eng._ctx, 1, None, C.c_int64(0), None, None) == 0
        assert eng._l.mvicp_closest_points(eng._ctx, 1, None, C.c_int64(0), None, None) == 0
        assert eng._l.mvicp_closest_points_device(eng._ctx, 2, _vp(q), C.c_int64(len(q)), _vp(idx), _vp(d2)) == INVALID
        assert eng._l.mvicp_closest_points(eng._ctx, -1, _vp(q), C.c_int64(len(q)), _vp(idx), _vp(d2)) == INVALID
        eng.close()


def test_set_edge_device_twin(emu):
    """mvicp_set_edge_device leaves what mvicp_set_edge leaves: duplicates (last occurrence wins), count as given, the next
    optimize's poses; an out-of-range index is refused and the edge stays as it was."""
    from mv_lm_icp_b200 import Engine, synth
    sc = _scene()
    edges = synth.ring_edges(3, 2)
    engs = []
    for _ in range(2):
        eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges); eng.set_poses(sc["poses_init"])
        eng.correspond(0.05)
        engs.append(eng)
    rng = np.random.default_rng(11)
    e = next(i for i, (s, _) in enumerate(edges) if s != 0)
    n_src, n_dst = engs[0].n_pts[edges[e][0]], engs[0].n_pts[edges[e][1]]
    first = rng.integers(0, n_src, 300).astype(np.int32)
    first[50:60] = first[10]                            # duplicates: the last of them wins
    second = rng.integers(0, n_dst, 300).astype(np.int32)
    engs[0].set_edge(e, first, second, 0.25)
    f, s = first.copy(), second.copy()
    assert engs[1]._l.mvicp_set_edge_device(engs[1]._ctx, C.c_int32(e), _vp(f), _vp(s), C.c_int64(300), C.c_float(0.25)) == 0
    before = engs[1].get_edge(e)
    assert all(np.array_equal(x, y) for x, y in zip(engs[0].get_edge(e), before))
    assert engs[0].get_edge(e, arrays=False) == engs[1].get_edge(e, arrays=False) == (300, np.float32(0.25))
    bad = first.copy(); bad[123] = n_src
    assert engs[1]._l.mvicp_set_edge_device(engs[1]._ctx, C.c_int32(e), _vp(bad), _vp(s), C.c_int64(300), C.c_float(0.5)) == INVALID
    assert b"at 123" in engs[1]._l.mvicp_last_error()
    bad2 = second.copy(); bad2[7] = -1
    assert engs[1]._l.mvicp_set_edge_device(engs[1]._ctx, C.c_int32(e), _vp(f), _vp(bad2), C.c_int64(300), C.c_float(0.5)) == INVALID
    after = engs[1].get_edge(e)
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    assert engs[1].get_edge(e, arrays=False) == (300, np.float32(0.25))
    assert engs[1]._l.mvicp_set_edge_device(engs[1]._ctx, C.c_int32(len(edges)), _vp(f), _vp(s), C.c_int64(3), C.c_float(0.5)) == INVALID
    for g in engs:
        g.optimize()
    Pa, Pb = (g.get_poses() for g in engs)
    assert Pa.tobytes() == Pb.tobytes()
    # an empty list resets the edge, as the host twin does
    engs[0].set_edge(e, np.zeros(0, np.int32), np.zeros(0, np.int32), 1.0)
    assert engs[1]._l.mvicp_set_edge_device(engs[1]._ctx, C.c_int32(e), None, None, C.c_int64(0), C.c_float(1.0)) == 0
    assert engs[0].get_edge(e, arrays=False) == engs[1].get_edge(e, arrays=False) == (0, np.float32(1.0))
    assert len(engs[1].get_edge(e)[0]) == 0
    for g in engs:
        g.close()


def test_normals_and_knn_self_twins(emu):
    from mv_lm_icp_b200 import Engine
    sc = _scene()
    eng = Engine(); eng.set_frames(sc["pts"], None)
    out = np.zeros((eng.n_pts[1], 3))
    assert eng._l.mvicp_get_normals_device(eng._ctx, 1, _vp(out)) == STATE
    nor, _ = eng.recompute_normals(10)
    for f in range(eng.M):
        out = np.zeros((eng.n_pts[f], 3))
        assert eng._l.mvicp_get_normals_device(eng._ctx, f, _vp(out)) == 0
        assert out.tobytes() == nor[f].tobytes()
    for k in (1, 10, 16):
        nn = np.full((eng.n_pts[2], k), -5, np.int32)
        assert eng._l.mvicp_knn_self_device(eng._ctx, 2, k, _vp(nn)) == 0
        assert np.array_equal(nn, eng.knn_self(2, k))
    assert eng._l.mvicp_knn_self_device(eng._ctx, 2, 0, _vp(nn)) == INVALID
    assert eng._l.mvicp_knn_self_device(eng._ctx, 3, 10, _vp(nn)) == INVALID
    eng.close()
