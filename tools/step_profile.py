"""Development aid: per-phase clock64() cycles of lm_step_kernel's launches in a one-problem solve (MVICP_STEP_PROFILE=1; the
joint optimize, or a component solve with one free component).  usage (GPU box):
MVICP_STEP_PROFILE=1 python tools/step_profile.py [views] [points]
With max_num_iterations = 1 a solve is two launches: #1 takes the initial evaluation, builds and factors the system and makes the
candidate; #2 takes the candidate's evaluation, accepts or rejects it and stops."""
import ctypes as C, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["MVICP_STEP_PROFILE"] = "1"
import mv_lm_icp_b200 as mv
from mv_lm_icp_b200 import synth, _lib
from mv_lm_icp_b200.api import default_options
M = int(sys.argv[1]) if len(sys.argv) > 1 else 20; N = int(sys.argv[2]) if len(sys.argv) > 2 else 20000
sc = synth.make_scene(M, N, config_id=3)
eng = mv.Engine(); eng.set_frames(sc["pts"], sc["nor"]); eng.set_graph(synth.ring_edges(M, 2)); eng.set_poses(sc["poses_init"])
opt = default_options(); opt.max_num_iterations = 1
names = ["wait+gather", "accept/take", "diag+build", "cholesky", "mcc+candidate", "writeback", "flag"]
for rnd in range(3):
    eng.correspond(0.05); eng.optimize(mv.PARAM_SE3, mv.COST_P2PLANE, True, opt)
    p = np.zeros(64, np.int64)
    _lib.check(_lib.lib().mvicp_debug_step_profile(eng._ctx, p.ctypes.data_as(C.POINTER(C.c_longlong))))
    for launch in (1, 2):
        q = p[16 * launch: 16 * launch + 16]
        if launch == 1:
            d = np.diff(q[:8])
            print(f"views {M} round {rnd} launch 1: total {q[7] - q[0]} cycles; " + ", ".join(f"{n} {v}" for n, v in zip(names, d))
                  + f"; inside cholesky: panel {q[8]} look-ahead/update {q[9]} barriers {q[10]}")
        else:
            print(f"views {M} round {rnd} launch 2: total {q[7] - q[0]} cycles; wait+gather {q[1] - q[0]}, accept/take {q[2] - q[1]}, rest {q[7] - q[2]}")
