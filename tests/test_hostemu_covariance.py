"""The pose covariances (mvicp_covariance, cov_factor_kernel, cov_solve_kernel) compiled against the miniature CUDA model in
tools/hostemu and run through the small cases of tests/test_gpu_covariance.py on the CPU, with the threads of a CTA in ascending
and in random order.  This checks the host logic (components, fixed frames, pair classification, the read-out), the factor's
and the column solves' indexing over the skyline profiles and the independence of every block from the request list; the
hardware's roundings are covered by `pytest -m gpu`."""
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
        so2 = str(tmp_path_factory.mktemp("hostemu_cov") / "libmvicp_hostemu_random.so")
        shutil.copy(so, so2); so = so2
        os.environ["HOSTEMU_ORDER"] = "random"
    lib = C.CDLL(so); lib.mvicp_last_error.restype = C.c_char_p
    os.environ.pop("HOSTEMU_ORDER", None)
    lib.order = request.param
    saved = _lib._lib
    _lib._lib = lib
    yield lib
    _lib._lib = saved


def test_errors(emu):
    import test_gpu_covariance as T
    T.check_errors()


def test_ring_matches_oracle(emu, oracle):
    import test_gpu_covariance as T
    T.check_ring_grid(oracle, params=(T.PARAM_QUAT, T.PARAM_SE3), costs=(T.COST_MIXED,), robusts=(True,), n_points=300)


def test_hub_graph_matches_oracle(emu, oracle):
    import test_gpu_covariance as T
    M, edges, fixed = T.G.topology("hub_last")
    eng, pts, nor, fx = T.graph_engine(oracle, M, edges, fixed, n_points=300, views=T.G.HUB_RING)
    T.check_oracle(oracle, eng, pts, nor, edges, fx, T.PARAM_SE3, T.COST_P2PLANE, True, "hub_last")
    T.check_request_independence(eng, M)
    eng.close()


def test_batch_matches_fresh_engines(emu, oracle):
    import test_gpu_covariance as T
    comps = T.T.mixed_comps(oracle, n_points=300, wide=False)
    statuses = T.check_batch_cov(oracle, comps)
    assert statuses == {T.COV_OK, T.COV_FIXED, T.COV_INDEPENDENT, T.COV_SINGULAR}, statuses


def test_floating_component_is_singular(emu, oracle):
    import test_gpu_covariance as T
    T.check_floating_component(oracle, n_points=300)


def test_rank(emu):
    import test_gpu_covariance as T
    T.check_planar_patch(n=200)
    T.check_free_frame_without_inliers(n_points=300)


def test_calls_between_solves_change_nothing(emu, oracle):
    import test_gpu_covariance as T
    if emu.order != "ascending":
        pytest.skip("slow case: first pass only")
    T.check_no_side_effects(oracle, n_points=300)
