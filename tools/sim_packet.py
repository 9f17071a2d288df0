"""Packet-walk model of the far rounds (csrc/far.cuh) on top of tools/sim_search.cpp: the queries of a warp are 32 consecutive
positions of the src frame's tree order (one edge); per warp, warp-steps of the per-lane search run in lock step (the slowest
lane's step count: every trip of the loop costs one step for the whole warp) against warp-steps of one shared depth-first walk
(sim_packet).  Round 0: initial poses, no seeds; round 1: poses half-way to the truth, seeded by round 0's matches.  Both node
arrays: plain AABBs and the hybrid oriented boxes of the far rounds.  Same scene as tools/sim_run.py.
usage: g++ -O2 -std=c++17 -shared -fPIC -I$CUDA_HOME/include tools/sim_search.cpp -o /tmp/libsim.so
       python tools/sim_packet.py /tmp/libsim.so [warps]
Output (128 warps):
  round 0 (cold), AABBs                        lock step 165.2 (lane mean 135.7, type-aware 271.0) | packet 221.0 = 19.0 + 96.6 + 105.3 (17.6/32 lanes)
  round 1 (stale seeds), AABBs                 lock step 190.0 (lane mean 161.1, type-aware 318.8) | packet 252.8 = 21.4 + 111.2 + 120.2 (18.1/32)
  round 0 (cold), hybrid oriented boxes        lock step  96.6 (lane mean  79.8, type-aware 138.6) | packet 132.2 = 19.0 + 68.2 + 45.0 (17.1/32)
  round 1 (stale seeds), hybrid oriented boxes lock step 107.6 (lane mean  90.5, type-aware 158.0) | packet 141.2 = 21.3 + 74.7 + 45.2 (17.5/32)
i.e. the packet walk issues 1.31-1.37x the lock-step warp-steps (0.79-0.95x the type-aware count).  On the H100 it is nonetheless
2-3x faster in the far rounds (DESIGN.md 4.1): the model counts issue steps, not the scattered loads of the per-lane walk."""
import ctypes as C, sys, numpy as np
sys.path.insert(0, '.'); sys.path.insert(0, 'tests')
from mv_lm_icp_b200 import synth
from oracle import oracle as O

lib = C.CDLL(sys.argv[1] if len(sys.argv) > 1 else '/tmp/libsim.so')
W = int(sys.argv[2]) if len(sys.argv) > 2 else 128
lib.sim_build.restype = C.c_void_p
P64, PI = C.POINTER(C.c_double), C.POINTER(C.c_int)
M, N = 20, 200000
pts, gt, init = [], [], []
for v in (1, 2):
    p, n, P = synth.make_view(v, M, N, 0xB200 + 3000 + v); pts.append(p); gt.append(P)
    rng = np.random.default_rng(0xA000 + 3000 + v); Q = P.copy(); Q[:3, :3] = P[:3, :3] @ synth._so3_exp(rng.normal(0, .02, 3)); Q[:3, 3] += rng.normal(0, .01, 3); init.append(Q)
gt = np.stack(gt); init = np.stack(init)
src, dst = np.ascontiguousarray(pts[0]), np.ascontiguousarray(pts[1])
h = C.c_void_p(lib.sim_build(dst.ctypes.data_as(P64), C.c_int64(len(dst))))
hs = C.c_void_p(lib.sim_build(src.ctypes.data_as(P64), C.c_int64(len(src))))
order = np.zeros(N, np.int32); lib.sim_order(hs, order.ctypes.data_as(PI))
starts = np.random.default_rng(1).choice(N // 32, W, replace=False) * 32
ks = np.concatenate([order[s:s + 32] for s in starts])
kd = O.KdIndex(dst, 'kd')
buf = np.zeros(1 << 16, np.uint8); lib.sim_set_trace(buf.ctypes.data_as(C.POINTER(C.c_ubyte)), len(buf))


def run(name, poses, seed_idx):
    q = np.ascontiguousarray(O.edge_queries(pts[0][ks], poses[0], poses[1]))
    ri, _ = kd.closest_points(pts[0][ks], poses[0], poses[1], threads=8)
    sl = np.full(len(ks), -1, np.int32) if seed_idx is None else np.array([lib.sim_leaf_of(h, int(i)) for i in seed_idx], np.int32)
    lock = 0; typed = 0; lane_sum = 0; pk = (C.c_int64 * 4)(0, 0, 0, 0); out = np.zeros(32, np.int32); miss = 0
    for w in range(W):
        steps = []; main = []
        for j in range(32 * w, 32 * w + 32):
            cnt = (C.c_int64 * 4)(0, 0, 0, 0)
            r = lib.sim_query(h, q[j].ctypes.data_as(P64), int(sl[j]), 1, cnt)
            miss += int(r != ri[j]); steps.append(cnt[2])
            tr = buf[:lib.sim_trace_len()]; main.append(tr[(tr == 1) | (tr == 2)])
        lock += max(steps); lane_sum += sum(steps)
        # sim_warp.py's type-aware count: a trip of the main loop in which some lanes test boxes and others scan points issues both
        ml = max(len(m) for m in main)
        typed += max(s - len(m) for s, m in zip(steps, main)) + sum(len({m[i] for m in main if len(m) > i}) for i in range(ml))
        qq = np.ascontiguousarray(q[32 * w:32 * w + 32]); ss = np.ascontiguousarray(sl[32 * w:32 * w + 32])
        lib.sim_packet(h, qq.ctypes.data_as(P64), ss.ctypes.data_as(PI), 32, out.ctypes.data_as(PI), pk)
        miss += int(np.sum(out != ri[32 * w:32 * w + 32]))
    packet = (pk[0] + pk[1] + pk[2]) / W
    print('%-46s per lane, lock step %6.1f (lane mean %6.1f, type-aware %6.1f) | packet %6.1f = prologue %5.1f + node %5.1f + leaf %5.1f '
          '(lanes needing the step %4.1f/32) | packet / lock step %.2f, / type-aware %.2f | mismatches %d' %
          (name, lock / W, lane_sum / (32 * W), typed / W, packet, pk[0] / W, pk[1] / W, pk[2] / W, pk[3] / max(1, pk[1] + pk[2]), packet * W / lock, packet * W / typed, miss))
    return ri


print('%d warps of 32 queries, warp-steps per warp' % W)
half = init.copy(); half[:, :3, 3] = 0.5 * (init[:, :3, 3] + gt[:, :3, 3])
for obb in (0, 1):
    lib.sim_set_obb(h, obb)
    box = 'hybrid oriented boxes' if obb else 'AABBs'
    i0 = run('round 0 (cold), ' + box, init, None)
    run('round 1 (stale seeds), ' + box, half, i0)
