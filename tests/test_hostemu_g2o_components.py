"""The per-component g2o solve (mvicp_optimize_g2o_components: G2oGate, the one-CTA-per-problem g2o_step_kernel and its ticket)
compiled against the miniature CUDA model in tools/hostemu and run through small cases of tests/test_gpu_g2o_components.py on
the CPU, with the threads of a CTA in ascending and in random order.  This checks the logic of the batched state machine and the
skipping of finished problems; the hardware's roundings are covered by `pytest -m gpu`."""
import ctypes as C
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools", "hostemu"))


@pytest.fixture(scope="module", params=["ascending", "random"])
def emu(request, tmp_path_factory):
    """libmvicp_hostemu.so behind the ctypes binding for this module; the random pass loads a private copy with
    HOSTEMU_ORDER=random (read once when the library is loaded)."""
    import shutil
    import build_hostemu
    from mv_lm_icp_b200 import _lib
    so = build_hostemu.build()
    if request.param == "random":
        so2 = str(tmp_path_factory.mktemp("hostemu_g2o_cmp") / "libmvicp_hostemu_random.so")
        shutil.copy(so, so2); so = so2
        os.environ["HOSTEMU_ORDER"] = "random"
    lib = C.CDLL(so); lib.mvicp_last_error.restype = C.c_char_p
    os.environ.pop("HOSTEMU_ORDER", None)
    lib.order = request.param
    saved = _lib._lib
    _lib._lib = lib
    yield lib
    _lib._lib = saved


def test_api(emu):
    import test_gpu_g2o_components as T
    T.check_api(n_points=200)


def test_connected_graph_equals_optimize_g2o(emu, oracle):
    import test_gpu_g2o_components as T
    o = T.short_options(1, 3)
    T.check_connected(oracle, "ring_chord", costs=[T.COST_P2PLANE], paths=("nonrigid",), n_points=300, opts=o)


def test_batch_matches_fresh_engines(emu, oracle):
    """Pairs, a ring with a user-fixed frame whose out-edges carry matches, an all-fixed ring, an isolated frame and a free frame
    without inliers; the model bar is left to the GPU run."""
    import test_gpu_g2o_components as T
    from mv_lm_icp_b200 import synth
    kw = dict(n_points=250)
    comps = [T.Comp(oracle, 2, [(1, 0), (0, 1)], cfg=11, **kw),
             T.Comp(oracle, 5, synth.ring_edges(5, 2), fixed=(2,), cfg=14, **kw),
             T.Comp(oracle, 3, synth.ring_edges(3, 1), fixed=(0, 1, 2), cfg=15, **kw),
             T.Comp(oracle, 1, [], cfg=16, **kw),
             T.Comp(oracle, 4, [(1, 0), (2, 1), (1, 2), (2, 0), (3, 0)], empty=(4,), cfg=17, **kw)]
    T.check_batch(comps, T.COST_P2PLANE, T.short_options(2, 3), model=False)


def test_failed_factorisation_next_to_a_converging_pair(emu, oracle):
    import test_gpu_g2o_components as T
    o = T.default_g2o_options(); o.tau = 0.0; o.max_calls = 7; o.iterations_per_call = 1; o.max_trials = 3
    out = T.check_batch([T.failing_pair(), T.Comp(oracle, 2, [(1, 0)], cfg=21, n_points=250)], T.COST_P2P, o, model=False)
    assert out[0][0]["ended"] == T.END_NO_IMPROVEMENT and out[0][0]["accepted"] == 0, out[0][0]
