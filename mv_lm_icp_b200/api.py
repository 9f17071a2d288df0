"""Python host mirror of the reference's frame / optimiser interface, on top of the C ABI.

Reference names kept: Frame.{pts,nor,pose,fixed,neighbours}, Frame.computePoseNeighboursKnn,
Frame.computeClosestPointsToNeighbours (include/frame.h:38-55), ICP_Ceres.ceresOptimizer{,_ceresAngleAxis,_sophusSE3}
and the pairwise pointToPoint_* / pointToPlane_* (include/icp-ceres.h:30-42).

Per-point arrays may also be torch CUDA tensors (set_frames, set_edge, closest_points) and some results come back as tensors
(edges_device, get_normals_device, knn_self_device): those calls go through the C ABI's device twins, and the data never
visits the host.  torch is imported only on these paths."""
import collections
import contextlib
import ctypes as C
import sys

import numpy as np

from . import _lib
from ._lib import COV_FIXED, COV_INDEPENDENT, COV_OK, COV_SINGULAR, Config, G2oOptions, G2oSummary, LmOptions, LmSummary, Stats, check  # noqa: F401

PARAM_AA, PARAM_QUAT, PARAM_SE3 = 0, 1, 2
COST_P2P, COST_P2PLANE, COST_MIXED = 0, 1, 2
TERMINATION = ["FUNCTION_TOLERANCE", "GRADIENT_TOLERANCE", "PARAMETER_TOLERANCE", "MAX_ITERATIONS", "MIN_RADIUS",
               "INVALID_STEPS", "EVAL_FAILURE"]
FLAG_NO_SEED = 1
FLAG_NCCL_ONLY = 2
FLAG_HOST_BUILD = 4
FLAG_NO_ADJ = 8
FLAG_NO_OBB = 16
FLAG_STEP_LOOP = 32
FLAG_NO_SELECT_GUESS = 64
FLAG_NO_CERT = 128


def _p(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _pose16(P):
    return _f64(np.asarray(P, dtype=np.float64).T).reshape(16)   # column-major, as Isometry3d::data()


def _is_tensor(x):
    """A torch tensor, without importing torch: a caller who holds one has imported it already."""
    torch = sys.modules.get("torch")
    return torch is not None and isinstance(x, torch.Tensor)


def _vp(t):
    return C.c_void_p(t.data_ptr())


# edges_device(): first / second / dist are views into one buffer of 16-byte Correspondance records (frame.h:18-22); edge e's
# inliers are entries offsets[e] .. offsets[e + 1]; weights[e] = OutgoingEdge::weight
DeviceEdges = collections.namedtuple("DeviceEdges", "first second dist offsets weights")


def nccl_unique_id():
    buf = (C.c_char * 128)()
    check(_lib.lib().mvicp_nccl_unique_id(buf))
    return bytes(buf)


class Engine:
    """One mvicp_ctx (one GPU, one host thread at a time)."""

    def __init__(self, device=0, flags=0, stream=None):
        self._l = _lib.lib()
        self._ctx = C.c_void_p()
        self.device = device
        self._ext_stream = None
        stream = getattr(stream, "cuda_stream", stream)   # a torch.cuda.Stream, or a raw cudaStream_t handle
        cfg = Config(device, flags, stream)
        check(self._l.mvicp_create(C.byref(cfg), C.byref(self._ctx)))
        self.M = 0
        self.n_pts = []
        self._keep = None

    def _free_pinned(self):
        if getattr(self, "_rec_ptr", None) is not None and self._rec_ptr.value:
            self.host_edges = None; self._rec_buf = None
            self._l.mvicp_host_free(self._rec_ptr)
        self._rec_ptr = None

    def close(self):
        if self._ctx:
            self._free_pinned()
            self._l.mvicp_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- data ---------------------------------------------------------------------------------------
    def set_frames(self, pts, nor=None):
        """Frame::pts / Frame::nor of every frame: numpy-like arrays, or CUDA tensors [N, 3] (float32 or float64) on this engine's
        device, which never leave the device (mvicp_set_frames_device)."""
        if any(_is_tensor(p) for p in pts) or (nor is not None and any(_is_tensor(n) for n in nor)):
            return self._set_frames_device(pts, nor)
        M = len(pts)
        P = [_f64(p).reshape(-1, 3) for p in pts]
        N = None if nor is None else [None if n is None else _f64(n).reshape(-1, 3) for n in nor]
        PP = (C.POINTER(C.c_double) * M)(*[_p(p) for p in P])
        NN = None
        if N is not None:
            NN = (C.POINTER(C.c_double) * M)(*[(_p(n) if n is not None else None) for n in N])
        n = np.ascontiguousarray([len(p) for p in P], np.int64)
        check(self._l.mvicp_set_frames(self._ctx, C.c_int32(M), PP, NN, _p(n, C.c_int64)))
        self.M = M
        self.n_pts = [len(p) for p in P]

    def _set_frames_device(self, pts, nor):
        import torch
        if not all(_is_tensor(p) for p in pts) or (nor is not None and not all(n is None or _is_tensor(n) for n in nor)):
            raise TypeError("set_frames: mixing host arrays and tensors; pass every frame (and normal) the same way")
        P = [self._coords(p, "set_frames: pts[%d]" % i) for i, p in enumerate(pts)]
        N = None if nor is None else [None if n is None else self._coords(n, "set_frames: nor[%d]" % i) for i, n in enumerate(nor)]
        M = len(P)
        PP = (C.c_void_p * M)(*[p.data_ptr() for p in P])
        NN = None if N is None else (C.c_void_p * M)(*[(n.data_ptr() if n is not None else None) for n in N])
        n = np.ascontiguousarray([p.shape[0] for p in P], np.int64)
        with self._torch_stream():
            check(self._l.mvicp_set_frames_device(self._ctx, C.c_int32(M), PP, NN, _p(n, C.c_int64)))
        self.M = M
        self.n_pts = [int(p.shape[0]) for p in P]

    def _cuda(self, t, what):
        """t must be a CUDA tensor on this engine's device."""
        import torch
        if not _is_tensor(t) or t.device.type != "cuda":
            raise TypeError("%s: expected a CUDA tensor, got %s" % (what, t.device if _is_tensor(t) else type(t).__name__))
        if t.device.index != self.device:
            raise ValueError("%s: tensor on %s, engine on cuda:%d" % (what, t.device, self.device))
        return t

    def _coords(self, t, what):
        """[N, 3] float32 / float64 CUDA tensor -> contiguous float64 (widening float32 is exact), on torch's current stream."""
        import torch
        t = self._cuda(t, what)
        if t.ndim != 2 or t.shape[1] != 3 or t.dtype not in (torch.float32, torch.float64):
            raise TypeError("%s: expected [N, 3] float32 or float64, got %s %s" % (what, tuple(t.shape), t.dtype))
        return t.to(torch.float64).contiguous()

    @contextlib.contextmanager
    def _torch_stream(self):
        """The stream protocol of every tensor call: the engine's stream waits for torch's current stream before the call, and
        the current stream waits for the engine's stream after it -- so a tensor produced or consumed on the current stream needs
        no synchronisation by the caller.  An engine created on torch's current stream skips both waits."""
        import torch
        cur = torch.cuda.current_stream(self.device)
        h = self.stream()
        if cur.cuda_stream == h:
            yield
            return
        if self._ext_stream is None:
            self._ext_stream = torch.cuda.ExternalStream(h, device=torch.device("cuda", self.device))
        self._ext_stream.wait_stream(cur)
        try:
            yield
        finally:
            cur.wait_stream(self._ext_stream)

    def set_poses(self, poses, fixed=None):
        P = _f64(np.stack([_pose16(p) for p in poses]))
        fx = None if fixed is None else np.ascontiguousarray(fixed, np.uint8)
        check(self._l.mvicp_set_poses(self._ctx, _p(P), _p(fx, C.c_uint8) if fx is not None else None))

    def get_poses(self):
        P = np.zeros((self.M, 16))
        check(self._l.mvicp_get_poses(self._ctx, _p(P)))
        return np.stack([P[i].reshape(4, 4).T.copy() for i in range(self.M)])

    def set_graph(self, edges):
        E = len(edges)
        s = np.ascontiguousarray([e[0] for e in edges], np.int32)
        d = np.ascontiguousarray([e[1] for e in edges], np.int32)
        check(self._l.mvicp_set_graph(self._ctx, C.c_int32(E), _p(s, C.c_int32), _p(d, C.c_int32)))
        self.edges = [(int(a), int(b)) for a, b in edges]

    def pose_graph_knn(self, knn):
        check(self._l.mvicp_pose_graph_knn(self._ctx, C.c_int32(knn)))
        E = C.c_int32(0)
        check(self._l.mvicp_get_graph(self._ctx, C.byref(E), None, None))
        s = np.zeros(E.value, np.int32); d = np.zeros(E.value, np.int32)
        check(self._l.mvicp_get_graph(self._ctx, C.byref(E), _p(s, C.c_int32), _p(d, C.c_int32)))
        self.edges = list(zip(s.tolist(), d.tolist()))
        return self.edges

    # ---- hot path -----------------------------------------------------------------------------------
    def correspond(self, thresh=0.05):
        check(self._l.mvicp_correspond(self._ctx, C.c_float(thresh)))

    def get_edge(self, e, arrays=True):
        n = self.n_pts[self.edges[e][0]]
        cnt = C.c_int64(0); w = C.c_float(0)
        if not arrays:
            check(self._l.mvicp_get_edge(self._ctx, C.c_int32(e), None, None, None, C.byref(cnt), C.byref(w)))
            return cnt.value, np.float32(w.value)
        first = np.empty(n, np.int32); second = np.empty(n, np.int32); dist = np.empty(n, np.float64)
        check(self._l.mvicp_get_edge(self._ctx, C.c_int32(e), _p(first, C.c_int32), _p(second, C.c_int32), _p(dist),
                                     C.byref(cnt), C.byref(w)))
        c = cnt.value
        return first[:c].copy(), second[:c].copy(), dist[:c].copy(), np.float32(w.value)

    CORR_DTYPE = np.dtype([("first", np.int32), ("second", np.int32), ("dist", np.float64)])   # struct Correspondance (frame.h:18-22)

    def pull_all_edges(self, records=True):
        """Every edge's (first, second, dist) list and weight into host arrays, as Frame::computeClosestPointsToNeighbours
        leaves them in OutgoingEdge::correspondances (frame.cpp:158,176): one structured array + offsets (mvicp_get_all_edges).
        Returns the number of bytes that reached the host; self.host_edges[e] = (records view, weight)."""
        E = len(self.edges)
        off = np.zeros(E + 1, np.int64); w = np.zeros(E, np.float32)
        cap = sum(self.n_pts[s] for s, _ in self.edges)
        if records:
            if getattr(self, "_rec_buf", None) is None or len(self._rec_buf) < cap:
                self._free_pinned()
                ptr = C.c_void_p()
                check(self._l.mvicp_host_alloc(C.c_size_t(cap * self.CORR_DTYPE.itemsize), C.byref(ptr)))   # page-locked: the copy runs at link speed
                self._rec_ptr = ptr
                self._rec_buf = np.frombuffer((C.c_char * (cap * self.CORR_DTYPE.itemsize)).from_address(ptr.value), dtype=self.CORR_DTYPE) if cap else np.empty(0, self.CORR_DTYPE)
            check(self._l.mvicp_get_all_edges(self._ctx, self._rec_buf.ctypes.data_as(C.c_void_p), C.c_int64(cap), _p(off, C.c_int64), _p(w, C.c_float)))
            self.host_edges = [(self._rec_buf[off[e]:off[e + 1]], w[e]) for e in range(E)]
        else:
            check(self._l.mvicp_get_all_edges(self._ctx, None, C.c_int64(0), _p(off, C.c_int64), _p(w, C.c_float)))
            self.host_edges = [(None, w[e]) for e in range(E)]
        self.edge_offsets = off
        return int(off[E]) * 16 * int(records) + 4 * E + 8 * (E + 1)

    def edges_device(self):
        """Every edge's inliers as device tensors (mvicp_get_all_edges_device), without a host synchronisation: a DeviceEdges of
        first / second (int32) and dist (float64) -- views into one buffer of 16-byte records, valid up to offsets[E] -- offsets
        (int64, E + 1) and weights (float32, E).  Each call returns a fresh buffer: the next correspond does not touch it."""
        import torch
        dev = torch.device("cuda", self.device)
        E = len(self.edges)
        cap = sum(self.n_pts[s] for s, _ in self.edges)
        rec = torch.empty((cap, 4), dtype=torch.int32, device=dev)
        off = torch.empty(E + 1, dtype=torch.int64, device=dev); w = torch.empty(E, dtype=torch.float32, device=dev)
        with self._torch_stream():
            check(self._l.mvicp_get_all_edges_device(self._ctx, _vp(rec) if cap else None, C.c_int64(cap), _vp(off), _vp(w)))
        return DeviceEdges(rec[:, 0], rec[:, 1], rec.view(torch.float64)[:, 1], off, w)

    def get_nn(self, e):
        n = self.n_pts[self.edges[e][0]]
        idx = np.empty(n, np.int32); d2 = np.empty(n, np.float64)
        check(self._l.mvicp_get_nn(self._ctx, C.c_int32(e), _p(idx, C.c_int32), _p(d2)))
        return idx, d2

    def set_edge(self, e, first, second, weight):
        """OutgoingEdge::correspondances of edge e from (first, second) pairs: numpy-like arrays, or CUDA tensors (int32 / int64)
        that stay on the device (mvicp_set_edge_device)."""
        if _is_tensor(first) or _is_tensor(second):
            return self._set_edge_device(e, first, second, weight)
        f = np.ascontiguousarray(first, np.int32); s = np.ascontiguousarray(second, np.int32)
        check(self._l.mvicp_set_edge(self._ctx, C.c_int32(e), _p(f, C.c_int32), _p(s, C.c_int32), C.c_int64(len(f)),
                                     C.c_float(weight)))

    def _set_edge_device(self, e, first, second, weight):
        import torch
        f = self._cuda(first, "set_edge: first"); s = self._cuda(second, "set_edge: second")
        for t, what in ((f, "first"), (s, "second")):
            if t.ndim != 1 or t.dtype not in (torch.int32, torch.int64):
                raise TypeError("set_edge: %s must be a 1-D int32 or int64 tensor, got %s %s" % (what, tuple(t.shape), t.dtype))
        if f.shape[0] != s.shape[0]:
            raise ValueError("set_edge: first and second differ in length")
        if (f.dtype == torch.int64 or s.dtype == torch.int64) and 0 <= e < len(self.edges) and f.shape[0]:
            # the range check on the full values, before int32 narrowing could wrap e.g. 2^32 + 5 into range
            n_src, n_dst = self.n_pts[self.edges[e][0]], self.n_pts[self.edges[e][1]]
            bad = (f < 0) | (f >= n_src) | (s < 0) | (s >= n_dst)
            if bool(bad.any()):
                raise _lib.MvicpError(1, "set_edge: index out of range at %d" % int(bad.nonzero()[0, 0]))
        f = f.to(torch.int32).contiguous(); s = s.to(torch.int32).contiguous()
        with self._torch_stream():
            check(self._l.mvicp_set_edge_device(self._ctx, C.c_int32(e), _vp(f), _vp(s), C.c_int64(f.shape[0]), C.c_float(weight)))

    def closest_points(self, frame, q):
        """Frame::getClosestPoint for every row of q (frame-local coordinates), each bit for bit what closest_point returns; a
        non-finite query gets idx -1, d2 NaN.  A CUDA tensor [n, 3] (float32 / float64) gives (int64, float64) tensors and stays
        on the device; numpy gives numpy."""
        if _is_tensor(q):
            import torch
            q = self._coords(q, "closest_points: q")
            n = q.shape[0]
            idx = torch.empty(n, dtype=torch.int64, device=q.device); d2 = torch.empty(n, dtype=torch.float64, device=q.device)
            with self._torch_stream():
                check(self._l.mvicp_closest_points_device(self._ctx, C.c_int32(frame), _vp(q), C.c_int64(n), _vp(idx), _vp(d2)))
            return idx, d2
        q = _f64(q).reshape(-1, 3); n = len(q)
        idx = np.empty(n, np.int64); d2 = np.empty(n, np.float64)
        check(self._l.mvicp_closest_points(self._ctx, C.c_int32(frame), _p(q), C.c_int64(n), _p(idx, C.c_int64), _p(d2)))
        return idx, d2

    def closest_point(self, frame, q):
        q = _f64(q); idx = C.c_int64(0); d2 = C.c_double(0)
        check(self._l.mvicp_closest_point(self._ctx, C.c_int32(frame), _p(q), C.byref(idx), C.byref(d2)))
        return idx.value, d2.value

    def optimize(self, param=PARAM_SE3, cost=COST_P2PLANE, robust=True, options=None):
        s = LmSummary()
        check(self._l.mvicp_optimize(self._ctx, C.c_int32(param), C.c_int32(cost), C.c_int32(int(robust)),
                                     C.byref(options) if options is not None else None, C.byref(s)))
        return s.asdict()

    def components(self):
        """Connected components of the current graph (mvicp_get_components): (n, component_of_frame), numbered in ascending
        order of their lowest frame; a frame without edges is a component of its own."""
        n = C.c_int32(0); comp = np.zeros(self.M, np.int32)
        check(self._l.mvicp_get_components(self._ctx, C.byref(n), _p(comp, C.c_int32)))
        return n.value, comp

    def optimize_components(self, param=PARAM_SE3, cost=COST_P2PLANE, robust=True, options=None):
        """One independent LM solve per connected component, all in one batched loop (mvicp_optimize_components): each
        component ends exactly as optimize() would in an engine holding only that component.  Fixes the lowest frame of every
        component.  Returns one summary dict per component, in component order."""
        n = C.c_int32(0)
        check(self._l.mvicp_get_components(self._ctx, C.byref(n), None))
        s = (LmSummary * max(1, n.value))()
        check(self._l.mvicp_optimize_components(self._ctx, C.c_int32(param), C.c_int32(cost), C.c_int32(int(robust)),
                                                C.byref(options) if options is not None else None, s))
        return [s[k].asdict() for k in range(n.value)]

    def covariance(self, pairs=None, param=PARAM_SE3, cost=COST_P2PLANE, robust=True):
        """Covariance blocks of the problem optimize(param, cost, robust) would solve now, at the current poses
        (mvicp_covariance, ceres::Covariance in the parameterisation's tangent space): `pairs` is a list of (a, b) frame pairs,
        None for the diagonal block of every frame.  Returns (cov float64 [n, 6, 6], status int32 [n]) with cov[k] = Cov(x_a,
        x_b); status COV_OK, COV_FIXED (zeros), COV_INDEPENDENT (different components: zeros) or COV_SINGULAR (NaN)."""
        if pairs is None:
            pairs = [(f, f) for f in range(self.M)]
        p = np.asarray(pairs, np.int64).reshape(-1, 2)
        if p.size and (p.min() < -2**31 or p.max() >= 2**31):
            raise _lib.MvicpError(1, "covariance: frame index out of range")
        a = np.ascontiguousarray(p[:, 0], np.int32); b = np.ascontiguousarray(p[:, 1], np.int32)
        n = len(a)
        cov = np.zeros((n, 6, 6)); st = np.zeros(n, np.int32)
        check(self._l.mvicp_covariance(self._ctx, C.c_int32(param), C.c_int32(cost), C.c_int32(int(robust)), C.c_int32(n),
                                       _p(a, C.c_int32), _p(b, C.c_int32), _p(cov), _p(st, C.c_int32)))
        return cov, st

    def icp_round(self, thresh=0.05, param=PARAM_SE3, cost=COST_P2PLANE, robust=True, options=None):
        s = LmSummary()
        check(self._l.mvicp_icp_round(self._ctx, C.c_float(thresh), C.c_int32(param), C.c_int32(cost),
                                      C.c_int32(int(robust)), C.byref(options) if options is not None else None, C.byref(s)))
        return s.asdict()

    def optimize_g2o(self, cost=COST_P2PLANE, options=None):
        """ICP_G2O::g2oOptimizer on the stored correspondences (icp-g2o.cpp:149-303): (summary dict, chi2 before the first call
        and after every call)."""
        o = options if options is not None else default_g2o_options()
        s = G2oSummary(); chi = np.zeros(o.max_calls + 1)
        check(self._l.mvicp_optimize_g2o(self._ctx, C.c_int32(cost), C.byref(o), C.byref(s), _p(chi)))
        d = s.asdict()
        return d, chi[:d["calls"] + 1].copy()

    def optimize_g2o_components(self, cost=COST_P2PLANE, options=None):
        """One independent g2o solve per connected component, all in one batched loop (mvicp_optimize_g2o_components): each
        component ends exactly as optimize_g2o() would in an engine holding only that component.  Fixes the lowest frame of
        every component.  Returns one (summary dict, chi2 before the first call and after every call) per component, in
        component order."""
        o = options if options is not None else default_g2o_options()
        n = C.c_int32(0)
        check(self._l.mvicp_get_components(self._ctx, C.byref(n), None))
        K = n.value
        s = (G2oSummary * max(1, K))(); chi = np.zeros((max(1, K), o.max_calls + 1))
        check(self._l.mvicp_optimize_g2o_components(self._ctx, C.c_int32(cost), C.byref(o), s, _p(chi)))
        out = []
        for k in range(K):
            d = s[k].asdict()
            out.append((d, chi[k, :d["calls"] + 1].copy()))
        return out

    def g2o_trace(self, component=None):
        """The last g2o solve's trials, one row each: lambda, chi, tchi, rho, accepted (mvicp_g2o_trace); with `component`,
        that component's trials of the last solve (mvicp_g2o_trace_component).  One row per trial run; rows past the recorded
        ones are zero."""
        n = C.c_int64(0)

        def fetch(out, cap):
            if component is None:
                return self._l.mvicp_g2o_trace(self._ctx, out, C.c_int64(cap), C.byref(n))
            return self._l.mvicp_g2o_trace_component(self._ctx, C.c_int32(component), out, C.c_int64(cap), C.byref(n))
        check(fetch(None, 0))
        out = np.zeros((n.value, 5))
        if n.value:
            check(fetch(_p(out), n.value))
        return out

    def recompute_normals(self, k=10, fetch=True):
        """Frame::recomputeNormals for every frame (frame.cpp:244-255). Returns (list of [N,3] normals, device ms);
        fetch=False leaves the normals on the device (list is None)."""
        check(self._l.mvicp_recompute_normals(self._ctx, C.c_int32(k)))
        out = []; ms = C.c_float(0)
        if not fetch:
            nor = np.empty((self.n_pts[0], 3))
            check(self._l.mvicp_get_normals(self._ctx, C.c_int32(0), _p(nor), C.byref(ms)))
            return None, ms.value
        for f in range(self.M):
            nor = np.empty((self.n_pts[f], 3))
            check(self._l.mvicp_get_normals(self._ctx, C.c_int32(f), _p(nor), C.byref(ms)))
            out.append(nor)
        return out, ms.value

    def knn_self(self, frame, k=10):
        """Frame::getNeighbours for every point of a frame (frame.cpp:208-242): int32 [N, k]."""
        nn = np.empty((self.n_pts[frame], k), np.int32)
        check(self._l.mvicp_knn_self(self._ctx, C.c_int32(frame), C.c_int32(k), _p(nn, C.c_int32)))
        return nn

    def get_normals_device(self, frame):
        """The recomputed normals of one frame as a float64 CUDA tensor [N, 3] (mvicp_get_normals_device)."""
        import torch
        out = torch.empty((self.n_pts[frame], 3), dtype=torch.float64, device=torch.device("cuda", self.device))
        with self._torch_stream():
            check(self._l.mvicp_get_normals_device(self._ctx, C.c_int32(frame), _vp(out)))
        return out

    def knn_self_device(self, frame, k=10):
        """knn_self as an int32 CUDA tensor [N, k] (mvicp_knn_self_device)."""
        import torch
        out = torch.empty((self.n_pts[frame], k), dtype=torch.int32, device=torch.device("cuda", self.device))
        with self._torch_stream():
            check(self._l.mvicp_knn_self_device(self._ctx, C.c_int32(frame), C.c_int32(k), _vp(out)))
        return out

    # ---- multi-GPU / introspection ---------------------------------------------------------------------
    def comm_init(self, unique_id, rank, world):
        check(self._l.mvicp_comm_init(self._ctx, C.c_char_p(unique_id), C.c_int32(rank), C.c_int32(world)))

    def stats(self):
        s = Stats()
        check(self._l.mvicp_get_stats(self._ctx, C.byref(s)))
        return s.asdict()

    def stream(self):
        p = C.c_void_p()
        check(self._l.mvicp_get_stream(self._ctx, C.byref(p)))
        return p.value

    def sync(self):
        check(self._l.mvicp_sync(self._ctx))


def default_options():
    o = LmOptions()
    _lib.lib().mvicp_default_lm_options(C.byref(o))
    return o


def default_g2o_options():
    o = G2oOptions()
    _lib.lib().mvicp_default_g2o_options(C.byref(o))
    return o


class OutgoingEdge:
    """include/frame.h:24-29"""

    def __init__(self, neighbourIdx, weight=0.0):
        self.neighbourIdx = neighbourIdx
        self.weight = np.float32(weight)
        self.correspondances = []   # list of (first, second, dist)


class Frame:
    """include/frame.h:31-102 (hot-path members only)."""

    def __init__(self, pts, nor=None, pose=None, fixed=False):
        self.pts = _f64(pts).reshape(-1, 3)
        self.nor = None if nor is None else _f64(nor).reshape(-1, 3)
        self.pose = np.eye(4) if pose is None else np.array(pose, dtype=np.float64)
        self.fixed = fixed
        self.neighbours = []

    # bound by ICP_Ceres / FrameSet below
    _engine = None
    _index = -1


class FrameSet:
    """A list of Frames sharing one Engine: the frame / correspondence plumbing that ICP_Ceres and ICP_G2O both stand on."""

    def __init__(self, frames, device=0, flags=0):
        self.frames = frames
        self.engine = Engine(device, flags)
        self.engine.set_frames([f.pts for f in frames], None if any(f.nor is None for f in frames) else [f.nor for f in frames])
        for i, f in enumerate(frames):
            f._engine, f._index = self.engine, i

    def _push_poses(self):
        self.engine.set_poses([f.pose for f in self.frames], [1 if f.fixed else 0 for f in self.frames])

    def _pull_poses(self):
        P = self.engine.get_poses()
        for i, f in enumerate(self.frames):
            f.pose = P[i]

    def recomputeNormals(self, k=10):   # Frame::recomputeNormals, main_multiview.cpp:68
        nor, _ = self.engine.recompute_normals(k)
        for f, n in zip(self.frames, nor):
            f.nor = n

    def computePoseNeighbours(self, knn):   # main_multiview.cpp:104-117
        self._push_poses()
        edges = self.engine.pose_graph_knn(knn)
        for f in self.frames:
            f.neighbours = []
        for s, d in edges:
            self.frames[s].neighbours.append(OutgoingEdge(d))
        return edges

    def computeClosestPoints(self, cutoff, materialize=False):   # main_multiview.cpp:119-127
        self._push_poses()
        self.engine.correspond(cutoff)
        if materialize:
            self.pull_correspondances()

    def pull_correspondances(self):
        e = 0
        for f in self.frames:
            for ne in f.neighbours:
                if f.fixed:
                    ne.correspondances = []
                else:
                    a, b, d, w = self.engine.get_edge(e)
                    ne.correspondances = list(zip(a.tolist(), b.tolist(), d.tolist())); ne.weight = w
                e += 1


class ICP_Ceres(FrameSet):
    """Drop-in for namespace ICP_Ceres (include/icp-ceres.h:22-45) over a list of Frames sharing one Engine."""

    def _opt(self, param, pointToPlane, robust, options=None):
        self.frames[0].fixed = True   # icp-ceres.cpp:242-244,342-344,417-419
        s = self.engine.optimize(param, COST_P2PLANE if pointToPlane else COST_P2P, robust, options)
        self._pull_poses()
        return s

    def ceresOptimizer(self, pointToPlane, robust, options=None):
        return self._opt(PARAM_QUAT, pointToPlane, robust, options)

    def ceresOptimizer_ceresAngleAxis(self, pointToPlane, robust, options=None):
        return self._opt(PARAM_AA, pointToPlane, robust, options)

    def ceresOptimizer_sophusSE3(self, pointToPlane, robust, automaticDiffLocalParam=True, options=None):
        return self._opt(PARAM_SE3, pointToPlane, robust, options)

    # ---- pairwise (include/icp-ceres.h:30-36) ------------------------------------------------------------
    @staticmethod
    def _pairwise(param, cost, src, dst, nor=None, device=0, options=None):
        src = _f64(src).reshape(-1, 3); dst = _f64(dst).reshape(-1, 3)
        nr = None if nor is None else _f64(nor).reshape(-1, 3)
        out = np.zeros(16); s = LmSummary(); cfg = Config(device, 0, None)
        check(_lib.lib().mvicp_pairwise(C.byref(cfg), C.c_int32(param), C.c_int32(cost), _p(src), _p(dst),
                                        _p(nr) if nr is not None else None, C.c_int64(len(src)),
                                        C.byref(options) if options is not None else None, _p(out), C.byref(s)))
        return out.reshape(4, 4).T.copy(), s.asdict()

    @staticmethod
    def closed_form(src, dst, nor=None, device=0):
        """ICP_Closedform::pointToPoint (nor is None) / pointToPlane (icp-closedform.cpp:9-54): 4x4 src -> dst."""
        src = _f64(src).reshape(-1, 3); dst = _f64(dst).reshape(-1, 3)
        nr = None if nor is None else _f64(nor).reshape(-1, 3)
        out = np.zeros(16); cfg = Config(device, 0, None)
        check(_lib.lib().mvicp_pairwise_closed(C.byref(cfg), C.c_int32(COST_P2P if nr is None else COST_P2PLANE), _p(src), _p(dst),
                                               _p(nr) if nr is not None else None, C.c_int64(len(src)), _p(out)))
        return out.reshape(4, 4).T.copy()

    @staticmethod
    def pointToPoint_EigenQuaternion(src, dst, **kw): return ICP_Ceres._pairwise(PARAM_QUAT, COST_P2P, src, dst, **kw)
    @staticmethod
    def pointToPoint_CeresAngleAxis(src, dst, **kw): return ICP_Ceres._pairwise(PARAM_AA, COST_P2P, src, dst, **kw)
    @staticmethod
    def pointToPoint_SophusSE3(src, dst, **kw): return ICP_Ceres._pairwise(PARAM_SE3, COST_P2P, src, dst, **kw)
    @staticmethod
    def pointToPlane_EigenQuaternion(src, dst, nor, **kw): return ICP_Ceres._pairwise(PARAM_QUAT, COST_P2PLANE, src, dst, nor, **kw)
    @staticmethod
    def pointToPlane_CeresAngleAxis(src, dst, nor, **kw): return ICP_Ceres._pairwise(PARAM_AA, COST_P2PLANE, src, dst, nor, **kw)
    @staticmethod
    def pointToPlane_SophusSE3(src, dst, nor, **kw): return ICP_Ceres._pairwise(PARAM_SE3, COST_P2PLANE, src, dst, nor, **kw)


class ICP_G2O(FrameSet):
    """Drop-in for namespace ICP_G2O (include/icp-g2o.h:9-15): g2oOptimizer over a FrameSet, and the two pairwise solvers."""

    def g2oOptimizer(self, pointToPlane, options=None):
        """icp-g2o.cpp:149-303: frame 0 becomes fixed, every frame's pose is written back.  Returns (summary, chi2 per call)."""
        self.frames[0].fixed = True   # icp-g2o.cpp:182-186
        self._push_poses()
        out = self.engine.optimize_g2o(COST_P2PLANE if pointToPlane else COST_P2P, options)
        self._pull_poses()
        return out

    @staticmethod
    def _pairwise_g2o(cost, src, dst, nor=None, device=0, options=None):
        src = _f64(src).reshape(-1, 3); dst = _f64(dst).reshape(-1, 3)
        nr = None if nor is None else _f64(nor).reshape(-1, 3)
        out = np.zeros(16); s = G2oSummary(); cfg = Config(device, 0, None)
        check(_lib.lib().mvicp_pairwise_g2o(C.byref(cfg), C.c_int32(cost), _p(src), _p(dst), _p(nr) if nr is not None else None,
                                            C.c_int64(len(src)), C.byref(options) if options is not None else None, _p(out),
                                            C.byref(s)))
        return out.reshape(4, 4).T.copy(), s.asdict()

    @staticmethod
    def pointToPoint(src, dst, **kw):
        """icp-g2o.cpp:26-85: the 4x4 pose of src in dst's frame, and the summary."""
        return ICP_G2O._pairwise_g2o(COST_P2P, src, dst, **kw)

    @staticmethod
    def pointToPlane(src, dst, nor, **kw):
        """icp-g2o.cpp:87-147 (nor: dst normals)."""
        return ICP_G2O._pairwise_g2o(COST_P2PLANE, src, dst, nor, **kw)
