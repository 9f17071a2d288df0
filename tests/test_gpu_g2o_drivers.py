"""The headless drivers' --g2o paths: apps/multiview_b200 on the reference's default 18 real frames against a CPU pipeline of
the oracle's correspondence step and the g2o restatement (tests/g2o_model.py), and apps/pairwise_b200's g2o accuracy row."""
import os
import re
import subprocess

import numpy as np
import pytest

import g2o_model as G
from helpers import host_threads, oracle_correspond, pose_rel_err
from test_gpu_real18 import _graph, _load

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_multiview_driver_g2o_matches_oracle_pipeline(oracle, golden_dir, tmp_path):
    """main_multiview.cpp --g2o (:158-164) on the 18 frames in the reference's on-disk formats, 2 rounds: the driver prints the
    reference's `round: s chi2:` / `round: k chi2: … impr: …` lines (icp-g2o.cpp:264,283-298) and ends within the 1e-5
    contract of the oracle's pipeline (own normals, own graph, own correspondences, g2o restatement)."""
    subprocess.run(["make", "-C", os.path.join(ROOT, "apps")], check=True, capture_output=True)
    pts, init, _ = _load(golden_dir)
    ids = list(range(0, 36, 2))
    for k, i in enumerate(ids):
        with open(tmp_path / f"cloudXYZ_{i}.xyz", "w") as f:
            for a in pts[k]:
                f.write("%.17g %.17g %.17g 0 0 1 \n" % tuple(a))
        np.savetxt(tmp_path / f"poses_{i}.txt", init[k], fmt="%.17g")
        with open(tmp_path / f"cloudXYZ_{i + 1}.xyz", "w") as f:
            f.write("0 0 0 0 0 1 \n")
        np.savetxt(tmp_path / f"poses_{i + 1}.txt", np.eye(4), fmt="%.17g")
    out = tmp_path / "out"; out.mkdir()
    R = 2
    r = subprocess.run([os.path.join(ROOT, "apps", "multiview_b200"), f"--dir={tmp_path}", "--sigma=0", "--sigmat=0", "--g2o",
                        f"--rounds={R}", f"--out={out}"], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    starts = re.findall(r"^round: s chi2: ([0-9.]+)$", r.stdout, flags=re.M)
    calls = re.findall(r"^round: (\d+) chi2: ([0-9.]+) impr: (\S+)$", r.stdout, flags=re.M)
    summ = [tuple(map(int, m)) for m in re.findall(r"^round: \d+  g2o calls (\d+) iterations (\d+) trials (\d+)", r.stdout, flags=re.M)]
    assert len(starts) == R and len(summ) == R and len(calls) == sum(c for c, _, _ in summ)
    got = np.stack([np.loadtxt(out / f"pose_out_{i}.txt") for i in range(18)])
    th = host_threads()
    nor = [oracle.recompute_normals(p, 10, threads=th) for p in pts]
    edges = _graph(oracle, init)
    poses = [P.copy() for P in init]
    for rnd in range(R):
        ref = oracle_correspond(oracle, pts, poses, edges, threads=th)
        corr = [((d["first"], d["second"]) if d else (np.zeros(0, np.int32), np.zeros(0, np.int32))) for d in ref]
        prob = G.Problem(pts, nor, edges, corr, [True] + [False] * 17, True)
        P, sm, chis, _ = G.optimize(prob, poses)
        assert abs(float(starts[rnd]) - chis[0]) <= 1e-6 + 1e-5 * chis[0], (rnd, starts[rnd], chis[0])   # printed with 6 decimals
        poses = list(P)
    assert pose_rel_err(got, np.stack(poses)) <= 1e-5, pose_rel_err(got, np.stack(poses))


@pytest.mark.parametrize("p2plane", [False, True])
def test_pairwise_driver_g2o_row(golden_dir, tmp_path, p2plane):
    """main_pairwise.cpp --g2o on cloud 0: the TIMING[g2o] line and the `g2o` accuracy row (:123-127), within the known-answer
    bounds 1e-10 m / 1e-6 degrees; the Ceres rows stay the last three."""
    subprocess.run(["make", "-C", os.path.join(ROOT, "apps")], check=True, capture_output=True)
    g = np.load(f"{golden_dir}/bunny_pair.npz")
    with open(tmp_path / "c.xyz", "w") as f:
        for a, n in zip(g["pts0"], g["nor0"]):
            f.write("%.17g %.17g %.17g %.17g %.17g %.17g\n" % (tuple(a) + tuple(n)))
    args = [os.path.join(ROOT, "apps", "pairwise_b200"), f"--cloud={tmp_path}/c.xyz", f"--out={tmp_path}", "--g2o"] + (["--pointToPlane"] if p2plane else [])
    r = subprocess.run(args, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert "=====  TIMING[g2o] is" in r.stdout
    m = re.findall(r"^g2o\s+\t diff_tra:([0-9.e+-]+)\t diff_rot_degrees:([0-9.e+-]+)", r.stdout, flags=re.M)
    assert len(m) == 1 and float(m[0][0]) <= 1e-10 and float(m[0][1]) < 1e-5, r.stdout
    rows = re.findall(r"diff_tra:([0-9.e+-]+)\t diff_rot_degrees", r.stdout)
    assert len(rows) == 5   # closed form, g2o, three Ceres rows
    P = np.loadtxt(tmp_path / "P_true.txt"); E = np.loadtxt(tmp_path / "P_g2o.txt")
    ang = np.degrees(np.linalg.norm(E[:3, :3] @ P[:3, :3].T - np.eye(3)) / np.sqrt(2))
    assert np.linalg.norm(E[:3, 3] - P[:3, 3]) <= 1e-10 and ang <= 1e-6, (E, P, ang)
