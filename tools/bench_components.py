"""Rate of the per-component solves (mvicp_optimize_components, mvicp_optimize_g2o_components): ICP rounds of correspond +
optimize_components (--solver lm) or correspond + optimize_g2o_components (--solver g2o) on a batch of independent
registrations, against one context per component run one after another, and against the joint optimize / optimize_g2o over
their union (a different problem: one trust region / one lambda for all; shown for time only).

  python tools/bench_components.py [--solver lm|g2o] [--workload pairs|real|3|all] [--rounds K] [--warmup W] [--reps R]
                                   [--pairs B] [--points N]

Workloads: `pairs` = B synthetic two-view problems of N points (8 distinct scenes, each pair from its own perturbed start);
`real` = the 18 Bunny_RealData frames of tests/golden/bunny18.npz (recomputed normals) cut into 9 pairs (2i, 2i + 1);
`3` = bench.py's config 3 (20 views x 200 k points, one component).  Point-to-plane, Sophus SE(3), robust, cutoff 0.05.  The
three arms alternate R times in one process; each run resets the poses, runs W rounds untimed and then K timed rounds (wall
clock between stream synchronisations).  The batched and the sequential arm must give the same poses per component: bit for bit
when the component's own context picks the batch's streaming tile length (the batch picks it from all components'
correspondence slots), else (LM) within 1e-12 relative; otherwise the tool exits with an error after its JSON line.  g2o's
rho > 0 and impr > 0 decisions are taken at rounding level near convergence (DESIGN section 2), so where the tile lengths differ
the g2o arms are only reported (largest relative pose and final chi2 difference), never failed.  g2o: the solver's defaults
(optimize(100) calls until noImpr passes 5).  Prints one JSON line with the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _rigid(rng, s_rot, s_tra):
    w = rng.normal(0, s_rot, 3); th = np.linalg.norm(w); k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    P = np.eye(4); P[:3, :3] = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K; P[:3, 3] = rng.normal(0, s_tra, 3)
    return P


NUM_SMS = 132        # csrc/types.cuh: the H100's SM count, which sizes the LM streaming tile
POSE_TOL = 1e-12     # relative pose difference allowed between the arms when their tile lengths differ


def tile_len(active):
    """The LM streaming tile mvicp.cu (layout_work) picks from the total of active correspondence slots."""
    tl = 8192
    while tl > 1024 and active // tl < 8 * NUM_SMS:
        tl >>= 1
    return tl


def active_slots(c):
    """Correspondence slots of a component's edges whose src is free (every frame but the lowest, here)."""
    return sum(len(c["pts"][s]) for s, _ in c["edges"] if s != 0)


def workload(name, n_pairs, n_points):
    """(list of components, each dict(pts, nor, poses, edges) in local frames; needs recomputed normals)"""
    import bench
    from mv_lm_icp_b200 import synth
    if name == "pairs":
        base = [synth.make_scene(2, n_points, config_id=500 + i) for i in range(min(8, n_pairs))]
        rng = np.random.default_rng(7)
        comps = []
        for i in range(n_pairs):
            b = base[i % len(base)]
            poses = b["poses_init"].copy(); poses[1] = _rigid(rng, 0.01, 0.005) @ poses[1]
            comps.append(dict(pts=b["pts"], nor=b["nor"], poses=poses, edges=[(0, 1), (1, 0)]))
        return comps, False
    cfg = bench.CONFIGS[name]
    sc = bench.load_scene(name, cfg)
    if name == "real":
        return [dict(pts=sc["pts"][2 * i:2 * i + 2], nor=None, poses=sc["poses_init"][2 * i:2 * i + 2].copy(), edges=[(0, 1), (1, 0)])
                for i in range(len(sc["pts"]) // 2)], True
    return [dict(pts=sc["pts"], nor=sc["nor"], poses=sc["poses_init"].copy(), edges=bench.scene_graph(sc, cfg))], sc["nor"][0] is None


def union(comps):
    """All components in one context: frames end to end, edges shifted."""
    pts, nor, poses, edges, first = [], [], [], [], []
    for c in comps:
        first.append(len(pts))
        edges += [(s + len(pts), d + len(pts)) for s, d in c["edges"]]
        pts += list(c["pts"]); nor += list(c["nor"]) if c["nor"] is not None else [None] * len(c["pts"]); poses += list(c["poses"])
    return dict(pts=pts, nor=nor if nor[0] is not None else None, poses=np.stack(poses), edges=edges), first


def engine(mv, c, recompute):
    eng = mv.Engine()
    eng.set_frames(c["pts"], c["nor"])
    if recompute:
        eng.recompute_normals(10, fetch=False)   # Frame::recomputeNormals (main_multiview.cpp:68)
    eng.set_graph(c["edges"])
    return eng


def run(engs, comps_of_eng, arm, rounds, warmup, mv, cutoff, solver="lm"):
    """One run of an arm: reset poses, warm up, time `rounds` rounds; returns (seconds, final poses per engine, g2o: the last
    round's final chi2 per component of every engine)."""
    for eng, c in zip(engs, comps_of_eng):
        fx = [0] * len(c["pts"])
        for f in c.get("lowest", [0]):
            fx[f] = 1
        eng.set_poses(c["poses"], fx)
    total = 0.0
    chi = [[] for _ in engs]
    for r in range(warmup + rounds):
        for eng in engs:
            eng.sync()
        t0 = time.perf_counter()
        for i, eng in enumerate(engs):
            eng.correspond(cutoff)
            if solver == "g2o" and arm == "batched":
                chi[i] = [s["chi2_final"] for s, _ in eng.optimize_g2o_components(mv.COST_P2PLANE)]
            elif solver == "g2o":
                chi[i] = [eng.optimize_g2o(mv.COST_P2PLANE)[0]["chi2_final"]]
            elif arm == "batched":
                eng.optimize_components(mv.PARAM_SE3, mv.COST_P2PLANE, True)
            else:
                eng.optimize(mv.PARAM_SE3, mv.COST_P2PLANE, True)
        for eng in engs:
            eng.sync()
        if r >= warmup:
            total += time.perf_counter() - t0
    return total, [eng.get_poses() for eng in engs], chi


def card():
    import torch
    name = torch.cuda.get_device_name(0) if torch.cuda.is_available() else None
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=20).stdout.strip()
    except Exception:
        pl = None
    return name, pl


def bench_workload(name, args):
    import bench
    import mv_lm_icp_b200 as mv
    comps, recompute = workload(name, args.pairs, args.points)
    u, first = union(comps)
    u_batched = dict(u, lowest=first)             # the batched context fixes every component's lowest frame
    engs = {"batched": [engine(mv, u, recompute)], "sequential": [engine(mv, c, recompute) for c in comps],
            "joint": [engine(mv, u, recompute)]}
    ctx = {"batched": [u_batched], "sequential": comps, "joint": [dict(u, lowest=first)]}
    times = {a: [] for a in engs}
    poses, chis = {}, {}
    for _ in range(args.reps):
        for arm in ("batched", "sequential", "joint"):
            t, P, chi = run(engs[arm], ctx[arm], arm, args.rounds, args.warmup, mv, bench.CUTOFF, args.solver)
            times[arm].append(t); poses[arm] = P; chis[arm] = chi
    # per component: bit for bit when its own context picks the batch's streaming tile, else within POSE_TOL (the tile fixes
    # how the edge sums are associated)
    Pb = poses["batched"][0]
    tl_batch = tile_len(sum(active_slots(c) for c in comps))
    diff, chi_diff, bitwise, ok, tiles = 0.0, 0.0, True, True, set()
    for k, (c, f0, Ps) in enumerate(zip(comps, first, poses["sequential"])):
        a, b = Pb[f0:f0 + len(c["pts"])], Ps
        same = np.array_equal(a.view(np.uint64), b.view(np.uint64))
        rel = float(np.max(np.abs(a - b)) / max(1.0, np.max(np.abs(b))))
        tl = tile_len(active_slots(c)); tiles.add(tl)
        if args.solver == "g2o":
            cb, cs = chis["batched"][0][k], chis["sequential"][k][0]
            same = same and np.float64(cb).view(np.uint64) == np.float64(cs).view(np.uint64)
            chi_diff = max(chi_diff, abs(cb - cs) / max(abs(cs), 1e-300))
            ok = ok and (same or tl != tl_batch)
        else:
            ok = ok and (same if tl == tl_batch else rel <= POSE_TOL)
        bitwise = bitwise and same
        diff = max(diff, rel)
    rate = {a: [round(args.rounds / t, 3) for t in ts] for a, ts in times.items()}
    for es in engs.values():
        for e in es:
            e.close()
    agree = {"ok": bool(ok), "bitwise": bool(bitwise), "max_rel_diff": diff, "tile_batched": tl_batch, "tile_sequential": sorted(tiles)}
    if args.solver == "g2o":
        agree["max_rel_chi2_diff"] = chi_diff
    return {"workload": name, "solver": args.solver, "components": len(comps), "frames": len(u["pts"]),
            "rounds_per_s": rate, "median_rounds_per_s": {a: float(np.median(v)) for a, v in rate.items()},
            "speedup_vs_sequential": float(np.median(rate["batched"]) / np.median(rate["sequential"])),
            "poses_batched_vs_sequential": agree}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solver", default="lm", choices=["lm", "g2o"])
    ap.add_argument("--workload", default="all", choices=["pairs", "real", "3", "all"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--points", type=int, default=20000)
    args = ap.parse_args()
    names = ["pairs", "real", "3"] if args.workload == "all" else [args.workload]
    gpu, power_limit = card()
    metric = {"lm": "correspond + optimize_components vs one context per component vs joint optimize",
              "g2o": "correspond + optimize_g2o_components vs one context per component vs joint optimize_g2o"}[args.solver]
    out = {"metric": "ICP rounds per second, " + metric,
           "gpu": gpu, "power_limit": power_limit, "rounds": args.rounds, "warmup": args.warmup, "reps": args.reps,
           "results": [bench_workload(n, args) for n in names]}
    print(json.dumps(out))
    if not all(r["poses_batched_vs_sequential"]["ok"] for r in out["results"]):
        sys.exit("bench_components: the batched and the sequential arm disagree on some component's poses")


if __name__ == "__main__":
    main()
