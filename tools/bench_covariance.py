"""Cost of the pose covariances (mvicp_covariance) next to the solve they describe: after K ICP rounds (correspond + optimize,
or + optimize_components on a batch) the call for the diagonal block of every frame is timed against one optimize
(optimize_components on a batch) from the same converged state.

  python tools/bench_covariance.py [--workload 3|pairs|all] [--rounds K] [--reps R] [--pairs B] [--points N]

Workloads (tools/bench_components.py): `3` = bench.py's config 3 (20 views x 200 k points, one component), `pairs` = B two-view
problems of N points in one context.  Point-to-plane, Sophus SE(3), robust, cutoff 0.05.  Each timed call ends in a stream
synchronisation (the covariance call returns its blocks on the host); the median of R repetitions is reported.  Prints one JSON
line with the card and its power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def bench_workload(name, args):
    import bench
    import bench_components as B
    import mv_lm_icp_b200 as mv
    comps, recompute = B.workload(name, args.pairs, args.points)
    u, first = B.union(comps)
    eng = B.engine(mv, u, recompute)
    batched = len(comps) > 1
    fx = [0] * len(u["pts"])
    for f in first:
        fx[f] = 1
    eng.set_poses(u["poses"], fx)

    def solve():
        return eng.optimize_components(mv.PARAM_SE3, mv.COST_P2PLANE, True) if batched else eng.optimize(mv.PARAM_SE3, mv.COST_P2PLANE, True)
    for _ in range(args.rounds):
        eng.correspond(bench.CUTOFF)
        solve()
    P = eng.get_poses()
    t_cov, t_opt = [], []
    cov, st = eng.covariance(None, mv.PARAM_SE3, mv.COST_P2PLANE, True)   # warm-up: layout upload, module load
    for _ in range(args.reps):
        eng.sync(); t0 = time.perf_counter()
        c2, s2 = eng.covariance(None, mv.PARAM_SE3, mv.COST_P2PLANE, True)
        t_cov.append(time.perf_counter() - t0)
        assert np.array_equal(c2.view(np.uint64), cov.view(np.uint64)) and np.array_equal(s2, st)
    solve()   # warm-up of the solve from this state
    for _ in range(args.reps):
        eng.set_poses(P, fx)
        eng.sync(); t0 = time.perf_counter()
        s = solve()
        eng.sync()
        t_opt.append(time.perf_counter() - t0)
    iters = max(x["num_iterations"] for x in s) if batched else s["num_iterations"]
    eng.close()
    counts = {k: int(np.sum(st == v)) for k, v in (("ok", mv.COV_OK), ("fixed", mv.COV_FIXED), ("singular", mv.COV_SINGULAR))}
    return {"workload": name, "components": len(comps), "frames": len(u["pts"]), "points": int(sum(len(p) for p in u["pts"])),
            "covariance_ms": round(1e3 * float(np.median(t_cov)), 3), "optimize_ms": round(1e3 * float(np.median(t_opt)), 3),
            "optimize_lm_iterations": int(iters), "ratio": round(float(np.median(t_cov) / np.median(t_opt)), 3), "status": counts}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="all", choices=["3", "pairs", "all"])
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--points", type=int, default=20000)
    args = ap.parse_args()
    import bench_components as B
    gpu, power_limit = B.card()
    names = ["3", "pairs"] if args.workload == "all" else [args.workload]
    out = {"metric": "mvicp_covariance (diagonal block of every frame) vs one optimize from the same converged state, median ms",
           "gpu": gpu, "power_limit": power_limit, "rounds": args.rounds, "reps": args.reps,
           "results": [bench_workload(n, args) for n in names]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
