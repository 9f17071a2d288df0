"""What it costs to use the correspondences and closest-point queries of the engine from the GPU (the C ABI's device twins,
include/mvicp.h), against the host-memory entry points.

  python tools/bench_device_io.py [--config 3|real|0|2] [--rounds K] [--reps R] [--queries N]

Workloads are bench.py's (same scenes, graph, cutoff, normals).  Three arms, alternated R times in one process, each K ICP rounds
from the initial poses (wall clock between stream synchronisations, rounds/s):
  1. icp_round alone (the correspondences stay inside the engine);
  2. correspond, pull_all_edges (every inlier record into page-locked host memory, mvicp_get_all_edges), optimize;
  3. correspond, edges_device (the records into a fresh CUDA tensor, mvicp_get_all_edges_device), optimize -- with a torch
     reduction over `dist` on the current stream, so that the records are really read.
The three arms must reach bit-identical poses.  Then closest-point queries against frame 0 of a synthetic workload (config 3: a
200 k-point frame): N queries near the surface (other frames' points, in frame 0's coordinates) and N uniform in the frame's
box, through mvicp_closest_points_device (tensors) and mvicp_closest_points (numpy), against 10^3 calls of the one-query entry
point mvicp_closest_point.  Prints one JSON line with the card's name and power limit (read, never set).  Writes nothing to the
repository (bench.py caches its synthetic scenes under /tmp)."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")[:2]]
        return name, limit
    except Exception:
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="3")
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--queries", type=int, default=1_000_000)
    args = ap.parse_args()
    import torch
    import bench
    import mv_lm_icp_b200 as mv
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_io: no CUDA device")
    cfg = bench.CONFIGS[args.config]
    sc = bench.load_scene(args.config, cfg)
    edges = bench.scene_graph(sc, cfg)
    param, cost = bench.PARAM[cfg["param"]], bench.COST[cfg["cost"]]
    eng = mv.Engine()
    eng.set_frames(sc["pts"], None if sc["nor"][0] is None else sc["nor"])
    if sc["nor"][0] is None:
        eng.recompute_normals(10, fetch=False)   # Frame::recomputeNormals (main_multiview.cpp:68)
    cur = torch.cuda.current_stream()
    acc = torch.zeros((), dtype=torch.float64, device="cuda")

    def arm(which, k):
        nonlocal acc
        eng.set_graph(edges); eng.set_poses(sc["poses_init"])
        torch.cuda.synchronize(); eng.sync()
        t0 = time.perf_counter()
        for _ in range(k):
            if which == 1:
                eng.icp_round(bench.CUTOFF, param, cost, True)
                continue
            eng.correspond(bench.CUTOFF)
            if which == 2:
                eng.pull_all_edges()
            else:
                d = eng.edges_device()
                valid = torch.arange(d.dist.shape[0], device="cuda") < d.offsets[-1]
                acc += torch.where(valid, d.dist, 0.0).sum()
            eng.optimize(param, cost, True)
        eng.sync(); cur.synchronize()
        dt = time.perf_counter() - t0
        return k / dt, hashlib.sha256(np.ascontiguousarray(eng.get_poses()).tobytes()).hexdigest()

    for w in (1, 2, 3):
        arm(w, 2)                                 # warm-up: module loads, buffers, pinned host memory
    rates = {1: [], 2: [], 3: []}; shas = {}
    for _ in range(args.reps):
        for w in (1, 2, 3):
            r, sha = arm(w, args.rounds)
            rates[w].append(r); shas[w] = sha
    records = int(eng.edge_offsets[-1])
    eng.close()

    out = {"metric": "ICP rounds per second with the correspondences used on the host / on the device", "config": args.config,
           "workload": bench.workload_name(args.config, cfg), "rounds": args.rounds, "reps": args.reps,
           "records_last_round": records, "record_bytes_last_round": 16 * records}
    for w, name in ((1, "icp_round"), (2, "pull_all_edges_host"), (3, "edges_device")):
        out[name] = {"rounds_per_s_median": float(np.median(rates[w])), "rounds_per_s": [round(x, 2) for x in rates[w]]}
    out["poses_equal_across_arms"] = len(set(shas.values())) == 1

    if not sc.get("real"):
        rng = np.random.default_rng(7)
        P = sc["poses_gt"]
        P0inv = np.linalg.inv(P[0])
        M, near, f = len(sc["pts"]), [], 0
        while sum(len(x) for x in near) < args.queries:   # frames 1, 2, ... in turn: their points in frame 0's local coordinates
            g = 1 + f % (M - 1); f += 1
            T = P0inv @ P[g]
            near.append(sc["pts"][g] @ T[:3, :3].T + T[:3, 3])
        near = np.ascontiguousarray(np.concatenate(near)[:args.queries])
        lo, hi = sc["pts"][0].min(0), sc["pts"][0].max(0)
        uni = np.ascontiguousarray(rng.uniform(lo, hi, (args.queries, 3)))
        e = mv.Engine(); e.set_frames([sc["pts"][0]], None)
        q_one = near[rng.choice(args.queries, 1000, replace=False)]
        e.closest_point(0, q_one[0])
        t0 = time.perf_counter()
        for q in q_one:
            e.closest_point(0, q)
        single = len(q_one) / (time.perf_counter() - t0)
        qs = {}
        for name, q in (("near_surface", near), ("uniform_box", uni)):
            qt = torch.from_numpy(q).cuda()
            e.closest_points(0, qt); e.closest_points(0, q[:1000])   # warm-up
            dev, host = [], []
            for _ in range(5):
                torch.cuda.synchronize(); t0 = time.perf_counter()
                i_d, d_d = e.closest_points(0, qt)
                torch.cuda.synchronize(); dev.append(len(q) / (time.perf_counter() - t0))
                t0 = time.perf_counter()
                i_h, d_h = e.closest_points(0, q)
                host.append(len(q) / (time.perf_counter() - t0))
            same = bool(np.array_equal(i_d.cpu().numpy(), i_h) and d_d.cpu().numpy().tobytes() == d_h.tobytes())
            qs[name] = {"device_queries_per_s": float(np.median(dev)), "host_queries_per_s": float(np.median(host)),
                        "device_equals_host": same}
        e.close()
        out["closest_points"] = {"frame_points": len(sc["pts"][0]), "queries": args.queries, "single_query_per_s": single, **qs}
    name, limit = card()
    out["gpu"] = name or torch.cuda.get_device_name(0)
    out["power_limit"] = limit
    out["checksum_dist_sum"] = float(acc.item())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
