"""Rate of the g2o backend (mvicp_optimize_g2o; icp-g2o.cpp): ICP rounds of closest points + g2oOptimizer, as main_multiview.cpp
runs them with --g2o (:150-169).

  python tools/bench_g2o.py [--config 3|real|0|2] [--rounds K] [--warmup W] [--cost p2plane|p2p]

Workloads are bench.py's (same scenes, graph, cutoff, normals): config 3 = 20 synthetic views x 200 k points, `real` = the 18
Bunny_RealData frames with recomputed normals.  After W warm-up rounds the poses are reset and K rounds are timed one by one
(wall clock between stream synchronisations).  Prints one JSON line: rounds/s, and per round the wall time, the g2o calls,
iterations and trials, the chi2 before and after, and the device time of the streaming kernels against the rest of the
solve.  Writes nothing to the repository (bench.py caches its synthetic scenes under /tmp)."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="3")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cost", default="p2plane", choices=["p2plane", "p2p"])
    args = ap.parse_args()
    import bench
    import mv_lm_icp_b200 as mv
    cfg = bench.CONFIGS[args.config]
    sc = bench.load_scene(args.config, cfg)
    edges = bench.scene_graph(sc, cfg)
    cost = mv.COST_P2PLANE if args.cost == "p2plane" else mv.COST_P2P
    eng = mv.Engine()
    eng.set_frames(sc["pts"], None if sc["nor"][0] is None else sc["nor"])
    if sc["nor"][0] is None:
        eng.recompute_normals(10, fetch=False)   # Frame::recomputeNormals (main_multiview.cpp:68)
    eng.set_graph(edges)

    def run(k, timed):
        eng.set_poses(sc["poses_init"])
        rows = []
        for _ in range(k):
            eng.sync(); t0 = time.perf_counter()
            eng.correspond(bench.CUTOFF)
            s, chi = eng.optimize_g2o(cost)
            eng.sync(); dt = time.perf_counter() - t0
            if timed:
                st = eng.stats()
                rows.append(dict(wall_ms=round(1e3 * dt, 3), calls=s["calls"], iterations=s["iterations"], trials=s["trials"],
                                 accepted=s["accepted"], evaluations=s["evaluations"], chi2_initial=s["chi2_initial"],
                                 chi2_final=s["chi2_final"], correspond_ms=round(st["correspond_ms"], 3),
                                 g2o_eval_ms=round(st["lm_eval_ms"], 3), g2o_other_ms=round(st["lm_other_ms"], 3)))
        return rows

    run(args.warmup, False)
    rows = run(args.rounds, True)
    import torch
    total = sum(r["wall_ms"] for r in rows) * 1e-3
    print(json.dumps({"metric": "g2o ICP rounds per second", "config": args.config, "workload": bench.workload_name(args.config, cfg),
                      "cost": args.cost, "rounds": len(rows), "rounds_per_s": len(rows) / total if total > 0 else None,
                      "median_round_ms": float(np.median([r["wall_ms"] for r in rows])) if rows else None,
                      "gpu": torch.cuda.get_device_name(0) if torch.cuda.is_available() else None, "per_round": rows}))
    eng.close()


if __name__ == "__main__":
    main()
