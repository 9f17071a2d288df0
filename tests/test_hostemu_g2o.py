"""The g2o backend's device code (g2o.cuh and its host loop in mvicp.cu) compiled against the miniature CUDA model in tools/hostemu
and run through the small parity cases of tests/test_gpu_g2o.py on the CPU, as tests/test_hostemu_engine.py does for the
Ceres-style path.  This checks the logic of the streaming kernel, the per-edge reduction and the LM state machine; the
hardware's roundings are covered by `pytest -m gpu`."""
import ctypes as C
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools", "hostemu"))


@pytest.fixture(scope="module")
def emu():
    import build_hostemu
    from mv_lm_icp_b200 import _lib
    lib = C.CDLL(build_hostemu.build()); lib.mvicp_last_error.restype = C.c_char_p
    saved = _lib._lib
    _lib._lib = lib
    yield lib
    _lib._lib = saved


@pytest.mark.parametrize("cost", [0, 1])
@pytest.mark.parametrize("fp64,nonrigid", [(False, False), (True, True)])
def test_ring(emu, cost, fp64, nonrigid):
    import test_gpu_g2o as T
    T.test_ring_matches_model(cost, fp64, nonrigid, n_views=3, n_points=400)


def test_loop_closure_and_empty_frame(emu):
    import test_gpu_g2o as T
    T.test_loop_closure_second_fixed_frame_and_an_empty_frame(1, n_points=300)


def test_options_and_errors(emu):
    import test_gpu_g2o as T
    T.test_options_and_errors()


@pytest.mark.parametrize("ortho_after", [1000, 2])
def test_rejected_trials_and_orthonormalisation(emu, ortho_after):
    import test_gpu_g2o as T
    T.test_rejected_trials_and_orthonormalisation(ortho_after)


def test_non_unit_normals(emu):
    import test_gpu_g2o as T
    T.test_non_unit_normals(1.3, n_views=3, n_points=400)
