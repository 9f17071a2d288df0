"""Per-point data that stays on the GPU: the C ABI's device twins (include/mvicp.h) through the Python API's torch tensor paths.
Every twin must return the same bytes as its host-memory counterpart: uploads (every storage mode, device and host tree build),
the correspondence export, batched closest-point queries, caller-supplied matches, normals and k-NN lists.  Also the stream
protocol (no manual synchronisation around a tensor call), the pointer check, and that the export does not wait for the
device."""
import ctypes as C
import os

import numpy as np
import pytest

from mv_lm_icp_b200 import COST_P2P, COST_P2PLANE, Engine, MvicpError, synth
from mv_lm_icp_b200.api import default_options

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAG_HOST_BUILD = 4
INVALID, STATE = 1, 4
CERTIFIED = []   # cert_rounds of every upload-twin run: at least one of them must have certified rounds


def _bunny(golden_dir):
    z = np.load(f"{golden_dir}/bunny18.npz")
    off = z["offsets"]; xyz = z["xyz_e8"].astype(np.float64) / 1e8
    return [np.ascontiguousarray(xyz[off[i]:off[i + 1]]) for i in range(int(z["n_frames"]))], z["poses_init"]


def _graph(poses):
    edges = []
    for i in range(len(poses)):
        d = sorted(((np.float32(np.linalg.norm(poses[i][:3, 3] - poses[j][:3, 3])), j) for j in range(len(poses)) if j != i), key=lambda x: x[0])
        edges += [(i, d[0][1]), (i, d[1][1])]
    return edges


def _host_edges(eng):
    eng.pull_all_edges()
    off = eng.edge_offsets.copy()
    return eng._rec_buf[:off[-1]].tobytes(), off, np.array([w for _, w in eng.host_edges], np.float32)


def _dev_edges(eng):
    d = eng.edges_device()
    off = d.offsets.cpu().numpy()
    n = int(off[-1])
    rec = torch.stack([d.first[:n], d.second[:n]], 1).cpu().numpy()
    dist = d.dist[:n].cpu().numpy()
    buf = np.zeros(n, Engine.CORR_DTYPE); buf["first"] = rec[:, 0]; buf["second"] = rec[:, 1]; buf["dist"] = dist
    return buf.tobytes(), off, d.weights.cpu().numpy()


def _same(a, b):
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2].view(np.uint32).tolist() == b[2].view(np.uint32).tolist()


STAT_KEYS = ("kernel_launches", "queries", "correspondences", "select_guess_rounds", "select_guess_misses", "cert_rounds", "cert_reused")


@pytest.mark.parametrize("flags", [0, FLAG_HOST_BUILD])
@pytest.mark.parametrize("mode", ["fp32_as_float32", "fp32_as_float64", "real_fp64", "p2p_no_normals", "recomputed_normals"])
def test_upload_twin(golden_dir, mode, flags):
    """An engine loaded from host arrays and one loaded from CUDA tensors (overwritten with NaN as soon as set_frames returns):
    bit-identical poses, edge lists and stats over 10 ICP rounds; the last five take one LM iteration each, so that the NN step
    reaches its certified rounds."""
    if mode == "real_fp64":
        pts, init = _bunny(golden_dir); nor = None; edges = _graph(init)
    else:
        sc = synth.make_scene(8, 20000, config_id=3)
        pts, init = sc["pts"], sc["poses_init"]
        nor = sc["nor"] if mode in ("fp32_as_float32", "fp32_as_float64") else None
        edges = synth.ring_edges(8, 2)
    dt = torch.float32 if mode == "fp32_as_float32" else torch.float64
    if dt == torch.float32:
        assert all(np.array_equal(p.astype(np.float32).astype(np.float64), p) for p in pts)   # exact in float32
    A = Engine(flags=flags); A.set_frames(pts, nor)
    B = Engine(flags=flags)
    P = [torch.tensor(p, dtype=dt, device="cuda") for p in pts]
    N = None if nor is None else [torch.tensor(n, dtype=dt, device="cuda") for n in nor]
    B.set_frames(P, N)
    for t in P + (N or []):
        t.fill_(float("nan"))
    cost = COST_P2P if mode == "p2p_no_normals" else COST_P2PLANE
    for eng in (A, B):
        if mode in ("recomputed_normals", "real_fp64"):
            eng.recompute_normals(10, fetch=False)
        eng.set_graph(edges); eng.set_poses(init)
    one = default_options(); one.max_num_iterations = 1
    for r in range(10):
        o = one if r >= 5 else None
        sa, sb = A.icp_round(0.05, cost=cost, options=o), B.icp_round(0.05, cost=cost, options=o)
        assert sa == sb, r
        assert A.get_poses().tobytes() == B.get_poses().tobytes(), r
        _same(_host_edges(A), _host_edges(B))
        ta, tb = A.stats(), B.stats()
        assert [ta[k] for k in STAT_KEYS] == [tb[k] for k in STAT_KEYS], r
    CERTIFIED.append(B.stats()["cert_rounds"])
    A.close(); B.close()


def test_some_upload_twin_run_was_certified():
    if not CERTIFIED:
        pytest.skip("run with test_upload_twin")
    assert max(CERTIFIED) > 0, CERTIFIED


def test_edge_export_equals_host_export():
    """edges_device after every round, byte for byte against mvicp_get_all_edges: an edge without inliers, a fixed src frame
    other than 0, NULL records; a capacity one below the bound and a call before correspond are refused."""
    sc = synth.make_scene(6, 20000, config_id=3)
    edges = synth.ring_edges(6, 2)
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(edges)
    eng.set_poses(sc["poses_init"])
    with pytest.raises(MvicpError) as ei:
        eng.edges_device()
    assert ei.value.code == STATE
    for r in range(6):
        eng.icp_round(0.05)
        eng.correspond(0.05)
        _same(_host_edges(eng), _dev_edges(eng))
    e = next(i for i, (s, _) in enumerate(edges) if s != 0)
    eng.set_edge(e, np.zeros(0, np.int32), np.zeros(0, np.int32), 0.0)                 # an edge without inliers
    _same(_host_edges(eng), _dev_edges(eng))
    fixed = np.zeros(6, np.uint8); fixed[3] = 1                                       # frame 3 fixed, frame 0 free
    eng.set_poses(eng.get_poses(), fixed); eng.correspond(0.05)
    h, d = _host_edges(eng), _dev_edges(eng)
    _same(h, d)
    assert all(d[1][i + 1] == d[1][i] for i, (s, _) in enumerate(edges) if s == 3)    # edges of the fixed frame: empty
    E = len(edges)
    off = torch.full((E + 1,), -1, dtype=torch.int64, device="cuda"); w = torch.zeros(E, dtype=torch.float32, device="cuda")
    assert eng._l.mvicp_get_all_edges_device(eng._ctx, None, C.c_int64(0), C.c_void_p(off.data_ptr()), C.c_void_p(w.data_ptr())) == 0
    eng.sync()
    assert np.array_equal(off.cpu().numpy(), h[1]) and w.cpu().numpy().tobytes() == h[2].tobytes()
    bound = sum(eng.n_pts[s] for s, _ in edges if s != 3)
    rec = torch.full((bound, 16), 0x5A, dtype=torch.uint8, device="cuda")
    off.fill_(-3)
    torch.cuda.synchronize()
    assert eng._l.mvicp_get_all_edges_device(eng._ctx, C.c_void_p(rec.data_ptr()), C.c_int64(bound - 1), C.c_void_p(off.data_ptr()), None) == INVALID
    eng.sync()
    assert bool((rec == 0x5A).all()) and bool((off == -3).all())
    assert eng._l.mvicp_get_all_edges_device(eng._ctx, C.c_void_p(rec.data_ptr()), C.c_int64(bound), C.c_void_p(off.data_ptr()), None) == 0
    eng.sync()
    assert rec.cpu().numpy()[:int(h[1][-1])].tobytes() == h[0]
    eng.close()


def test_edge_export_does_not_synchronise():
    """With the engine's stream held by a bounded sleep kernel, edges_device returns while that stream is still busy; the
    records are right once it has drained."""
    sc = synth.make_scene(4, 20000, config_id=3)
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(synth.ring_edges(4, 2)); eng.set_poses(sc["poses_init"])
    eng.correspond(0.05)
    ref = _host_edges(eng)
    es = torch.cuda.ExternalStream(eng.stream())
    with torch.cuda.stream(es):
        torch.cuda._sleep(200_000_000)        # ~0.1 s at H100 clocks
    d = eng.edges_device()
    busy = not es.query()
    eng.sync()
    assert busy
    off = d.offsets.cpu().numpy(); n = int(off[-1])
    assert np.array_equal(off, ref[1]) and d.weights.cpu().numpy().tobytes() == ref[2].tobytes()
    buf = np.zeros(n, Engine.CORR_DTYPE)
    buf["first"] = d.first[:n].cpu().numpy(); buf["second"] = d.second[:n].cpu().numpy(); buf["dist"] = d.dist[:n].cpu().numpy()
    assert buf.tobytes() == ref[0]
    eng.close()


def _brute(cloud, q):
    """Lowest index of the smallest (d0^2 + d1^2) + d2^2 (the reference's order), in fp64 on the GPU; each torch op rounds once."""
    P = torch.tensor(cloud, dtype=torch.float64, device="cuda")
    Q = torch.tensor(q, dtype=torch.float64, device="cuda")
    idx, d2 = [], []
    for a in range(0, len(Q), 256):
        d = Q[a:a + 256, None, :] - P[None, :, :]
        s = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        m = s.min(1).values
        first = (s == m[:, None]).int().argmax(1)
        idx.append(first); d2.append(m)
    return torch.cat(idx).cpu().numpy().astype(np.int64), torch.cat(d2).cpu().numpy()


@pytest.mark.parametrize("offset", [0.0, 1e5])
def test_closest_points_equal_single_query_and_brute_force(offset):
    """About 2000 queries of every kind, through the tensor and the numpy path: each equals mvicp_closest_point (index and d2
    bits) and a brute force in the reference's arithmetic; non-finite queries give -1 / NaN; n = 0; a bad frame."""
    sc = synth.make_scene(2, 20000, config_id=3)
    cloud = sc["pts"][1].copy()
    cloud[11] = cloud[5000]                                  # a duplicated point: ties go to index 11
    cloud = cloud + offset                                   # 1e5: not fp32-representable, fp64 storage
    rng = np.random.default_rng(2)
    size = float(np.max(cloud.max(0) - cloud.min(0)))
    ks = rng.integers(len(cloud), size=1500)
    q = np.concatenate([cloud[ks] + rng.normal(0, 0.002, (1500, 3)),          # on the surface
                        cloud.mean(0) + rng.normal(0, 1e3 * size, (200, 3)),  # far away
                        cloud[rng.integers(len(cloud), size=300)],            # exact copies
                        cloud[[11, 5000, 0]]])
    bad = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [np.nan] * 3])
    eng = Engine(); eng.set_frames([sc["pts"][0], cloud], None)
    qt = torch.tensor(np.concatenate([q, bad + offset]), device="cuda")
    it, dt = eng.closest_points(1, qt)
    it, dt = it.cpu().numpy(), dt.cpu().numpy()
    ih, dh = eng.closest_points(1, np.concatenate([q, bad + offset]))
    assert np.array_equal(it, ih) and it.dtype == np.int64 and dt.tobytes() == dh.tobytes()
    assert np.all(it[len(q):] == -1) and np.all(np.isnan(dt[len(q):]))
    it, dt = it[:len(q)], dt[:len(q)]
    bi, bd = _brute(cloud, q)
    assert np.array_equal(it, bi) and dt.tobytes() == bd.tobytes()
    for k in range(0, len(q), 7):
        i1, d1 = eng.closest_point(1, q[k])
        assert i1 == it[k] and np.float64(d1).tobytes() == dt[k].tobytes(), k
    assert it[-3] == 11 and it[-2] == 11 and dt[-2] == 0.0
    qf = torch.tensor(q, dtype=torch.float32, device="cuda")  # float32 queries are widened exactly
    i32, d32 = eng.closest_points(1, qf)
    ih32, dh32 = eng.closest_points(1, q.astype(np.float32).astype(np.float64))
    assert np.array_equal(i32.cpu().numpy(), ih32) and d32.cpu().numpy().tobytes() == dh32.tobytes()
    e0, d0 = eng.closest_points(1, torch.zeros((0, 3), dtype=torch.float64, device="cuda"))
    assert e0.shape == (0,) and d0.shape == (0,)
    with pytest.raises(MvicpError) as ei:
        eng.closest_points(2, qt)
    assert ei.value.code == INVALID
    eng.close()


def test_closest_points_million_queries():
    """10^6 queries against a 200 k-point frame, a 10 k sample against the brute force."""
    sc = synth.make_scene(2, 200_000, config_id=3)
    cloud = sc["pts"][0]
    T = np.linalg.inv(sc["poses_gt"][0]) @ sc["poses_gt"][1]
    near = sc["pts"][1] @ T[:3, :3].T + T[:3, 3]
    rng = np.random.default_rng(9)
    q = np.concatenate([near[rng.integers(len(near), size=700_000)], rng.uniform(cloud.min(0), cloud.max(0), (300_000, 3))])
    eng = Engine(); eng.set_frames([cloud], None)
    it, dt = eng.closest_points(0, torch.tensor(q, device="cuda"))
    s = rng.choice(len(q), 10_000, replace=False)
    bi, bd = _brute(cloud, q[s])
    assert np.array_equal(it.cpu().numpy()[s], bi) and dt.cpu().numpy()[s].tobytes() == bd.tobytes()
    eng.close()


@pytest.mark.parametrize("dtype", ["int32", "int64"])
def test_set_edge_from_tensors(dtype):
    """set_edge from CUDA tensors, with duplicates: get_edge and the next optimize's poses equal the host path's; an
    out-of-range index (also 2^32 + 5 for int64) is refused and leaves the edge unchanged."""
    sc = synth.make_scene(4, 20000, config_id=3)
    edges = synth.ring_edges(4, 2)
    engs = []
    for _ in range(2):
        g = Engine(); g.set_frames(sc["pts"], sc["nor"]); g.set_graph(edges); g.set_poses(sc["poses_init"]); g.correspond(0.05)
        engs.append(g)
    rng = np.random.default_rng(4)
    e = next(i for i, (s, _) in enumerate(edges) if s != 0)
    n_src, n_dst = engs[0].n_pts[edges[e][0]], engs[0].n_pts[edges[e][1]]
    first = rng.integers(0, n_src, 30000); first[100:200] = first[7]
    second = rng.integers(0, n_dst, 30000)
    engs[0].set_edge(e, first, second, 0.02)
    td = getattr(torch, dtype)
    ft, st = torch.tensor(first, dtype=td, device="cuda"), torch.tensor(second, dtype=td, device="cuda")
    engs[1].set_edge(e, ft, st, 0.02)
    a, b = engs[0].get_edge(e), engs[1].get_edge(e)
    assert all(np.asarray(x).tobytes() == np.asarray(y).tobytes() for x, y in zip(a, b))
    assert engs[0].get_edge(e, arrays=False) == engs[1].get_edge(e, arrays=False) == (30000, np.float32(0.02))
    bads = [n_src, -1] + ([2 ** 32 + 5] if dtype == "int64" else [])
    for v in bads:
        f2 = ft.clone(); f2[123] = v
        with pytest.raises(MvicpError) as ei:
            engs[1].set_edge(e, f2, st, 0.5)
        assert ei.value.code == INVALID and "123" in str(ei.value)
    s2 = st.clone(); s2[9] = n_dst
    with pytest.raises(MvicpError):
        engs[1].set_edge(e, ft, s2, 0.5)
    b2 = engs[1].get_edge(e)
    assert all(np.asarray(x).tobytes() == np.asarray(y).tobytes() for x, y in zip(b, b2))
    for g in engs:
        g.optimize()
    assert engs[0].get_poses().tobytes() == engs[1].get_poses().tobytes()
    for g in engs:
        g.close()


def test_normals_and_knn_self_device_twins():
    sc = synth.make_scene(3, 20000, config_id=3)
    eng = Engine(); eng.set_frames([torch.tensor(p, device="cuda") for p in sc["pts"]])
    with pytest.raises(MvicpError) as ei:
        eng.get_normals_device(0)
    assert ei.value.code == STATE
    nor, _ = eng.recompute_normals(10)
    for f in range(3):
        assert eng.get_normals_device(f).cpu().numpy().tobytes() == nor[f].tobytes()
    for k in (1, 10, 16):
        assert np.array_equal(eng.knn_self_device(1, k).cpu().numpy(), eng.knn_self(1, k))
    eng.close()


def test_stream_protocol():
    """An input produced on torch's current stream behind a sleep kernel is read correctly; an output is consumed right after
    the call without a synchronisation; an engine created on torch's stream works the same."""
    sc = synth.make_scene(3, 20000, config_id=3)
    rng = np.random.default_rng(6)
    q = sc["pts"][1][rng.integers(20000, size=50000)] + rng.normal(0, 0.003, (50000, 3))
    ref = Engine(); ref.set_frames(sc["pts"], sc["nor"])
    ri, rd = ref.closest_points(1, q)
    ref.close()
    s = torch.cuda.Stream()
    for on_torch_stream in (False, True):
        with torch.cuda.stream(s):
            eng = Engine(stream=s) if on_torch_stream else Engine()
            src = [torch.tensor(p, device="cuda") for p in sc["pts"]]
            torch.cuda._sleep(100_000_000)
            pts = [p * 1.0 for p in src]                     # written behind the sleep, on the current stream
            eng.set_frames(pts, [torch.tensor(n, device="cuda") for n in sc["nor"]])
            qa = torch.tensor(q, device="cuda")
            torch.cuda._sleep(100_000_000)
            qb = qa + 0.0
            idx, d2 = eng.closest_points(1, qb)
            total = (d2 * 1.0).sum()                          # consumed on the current stream, no synchronisation
            first = idx[:10].clone()
        torch.cuda.synchronize()
        assert np.array_equal(idx.cpu().numpy(), ri) and d2.cpu().numpy().tobytes() == rd.tobytes()
        assert np.array_equal(first.cpu().numpy(), ri[:10]) and float(total) == float(torch.tensor(rd, device="cuda").sum())
        if on_torch_stream:
            assert eng.stream() == s.cuda_stream
        eng.close()


def test_pointer_check():
    """A host pointer given to a device twin is refused before any work; a CPU tensor given to a tensor path raises; a tensor
    on another GPU is refused."""
    sc = synth.make_scene(2, 5000, config_id=3)
    eng = Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph([(1, 0)]); eng.correspond(0.05)
    q = np.zeros((4, 3)); idx = np.zeros(4, np.int64); d2 = np.zeros(4)
    vp = lambda a: C.c_void_p(a.ctypes.data)
    assert eng._l.mvicp_closest_points_device(eng._ctx, 0, vp(q), C.c_int64(4), vp(idx), vp(d2)) == INVALID
    off = np.zeros(2, np.int64)
    assert eng._l.mvicp_get_all_edges_device(eng._ctx, None, C.c_int64(0), vp(off), None) == INVALID
    f = np.zeros(3, np.int32)
    assert eng._l.mvicp_set_edge_device(eng._ctx, 0, vp(f), vp(f), C.c_int64(3), C.c_float(1.0)) == INVALID
    nn = np.zeros((5000, 10), np.int32)
    assert eng._l.mvicp_knn_self_device(eng._ctx, 0, 10, vp(nn)) == INVALID
    PP = (C.c_void_p * 1)(sc["pts"][0].ctypes.data); n = np.array([len(sc["pts"][0])], np.int64)
    assert eng._l.mvicp_set_frames_device(eng._ctx, 1, PP, None, n.ctypes.data_as(C.POINTER(C.c_int64))) == INVALID
    assert eng.get_poses().shape == (2, 4, 4)                # the refused upload left the frames as they were
    with pytest.raises(TypeError):
        eng.closest_points(0, torch.zeros((4, 3), dtype=torch.float64))
    with pytest.raises(TypeError):
        eng.set_frames([torch.zeros((4, 3), dtype=torch.float64), sc["pts"][1]])
    with pytest.raises(TypeError):
        eng.set_edge(0, torch.zeros(3, dtype=torch.int32), torch.zeros(3, dtype=torch.int32, device="cuda"), 1.0)
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            eng.closest_points(0, torch.zeros((4, 3), dtype=torch.float64, device="cuda:1"))
        x = torch.zeros((4, 3), dtype=torch.float64, device="cuda:1")
        r = eng._l.mvicp_closest_points_device(eng._ctx, 0, C.c_void_p(x.data_ptr()), C.c_int64(4), None, None)
        assert r == INVALID
    eng.close()


def test_tensor_on_another_gpu_is_rejected():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs a second GPU")
    sc = synth.make_scene(2, 5000, config_id=3)
    eng = Engine(device=0)
    with pytest.raises(ValueError):
        eng.set_frames([torch.tensor(p, device="cuda:1") for p in sc["pts"]])
    eng.close()
