"""The g2o backend's device code (g2o.cuh and its host loop in mvicp.cu) compiled against the miniature CUDA model in tools/hostemu
and run through the small parity cases of tests/test_gpu_g2o.py and tests/test_gpu_g2o_graphs.py on the CPU, as
tests/test_hostemu_engine.py does for the Ceres-style path.  This checks the logic of the streaming kernel, the per-edge
reduction and the LM state machine; the hardware's roundings are covered by `pytest -m gpu`."""
import ctypes as C
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools", "hostemu"))


@pytest.fixture(scope="module")
def _libs(tmp_path_factory):
    """libmvicp_hostemu.so loaded once per thread order.  "random": the threads of a CTA run in a fresh pseudo-random order
    between any two barriers (HOSTEMU_ORDER=random, read once when the library is loaded: a private copy is loaded)."""
    import shutil
    import build_hostemu
    from mv_lm_icp_b200 import _lib
    so = build_hostemu.build()
    libs = {}

    def get(order):
        if order not in libs:
            path = so
            if order == "random":
                path = str(tmp_path_factory.mktemp("hostemu_g2o") / "libmvicp_hostemu_random.so")
                shutil.copy(so, path)
                os.environ["HOSTEMU_ORDER"] = "random"
            lib = C.CDLL(path); lib.mvicp_last_error.restype = C.c_char_p
            os.environ.pop("HOSTEMU_ORDER", None)
            lib.order = order
            libs[order] = lib
        return libs[order]
    saved = _lib._lib
    yield get
    _lib._lib = saved


def _use(get, order):
    from mv_lm_icp_b200 import _lib
    saved = _lib._lib
    _lib._lib = get(order)
    return _lib, saved


@pytest.fixture
def emu(_libs):
    """The ctypes binding pointed at the host model (threads of a CTA in ascending order) for one test."""
    lib, saved = _use(_libs, "ascending")
    yield lib._lib
    lib._lib = saved


@pytest.fixture(params=["ascending", "random"])
def emu_pass(request, _libs):
    """As emu, in two passes: ascending and random thread order, so code that lacks a barrier cannot pass both; the slow
    cases run in the first pass only."""
    lib, saved = _use(_libs, request.param)
    yield lib._lib
    lib._lib = saved


def _first_pass_only(emu):
    if emu.order != "ascending":
        pytest.skip("slow case: first pass only")


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


def test_storage_modes(emu_pass, oracle):
    """Every storage mode, rigid and non-rigid poses, both costs (point-to-plane refused without normals)."""
    import test_gpu_g2o_graphs as T
    for mode in T.MODES:
        for path in ("unit", "general"):
            T.test_storage_modes_match_model(oracle, mode, path)


def test_graphs_and_fixed_sets(emu_pass, oracle):
    """Three topologies (the g2o-specific ones among them), every fixed set, all frames fixed, the fixed set switched."""
    import test_gpu_g2o_graphs as T
    for name in ("hub_last", "mid_empty", "fixed_src"):
        T.test_graph_topologies_match_model(oracle, name)
    for fixed in T.FIXED_SETS:
        T.test_fixed_sets_match_model(oracle, fixed)
    T.test_all_frames_fixed_leaves_poses_unchanged(oracle)


def test_switching_fixed_sets(emu_pass, oracle):
    import test_gpu_g2o_graphs as T
    _first_pass_only(emu_pass)
    T.test_switching_fixed_sets_between_solves(oracle)


def test_wide_graph_factor_in_global_memory(emu_pass, oracle):
    import test_gpu_g2o_graphs as T
    _first_pass_only(emu_pass)
    T.test_wide_graph_factor_in_global_memory(oracle, 48, True)


def test_tile_boundaries(emu_pass, oracle):
    import test_gpu_g2o_graphs as T
    T.test_tile_boundaries_chi2_readout(oracle, 1024)


@pytest.mark.parametrize("ortho_after", [1000, 2])
def test_failed_factorisation(emu_pass, ortho_after):
    import test_gpu_g2o_graphs as T
    T.test_failed_factorisation_is_a_rejected_trial(ortho_after)


def test_rotation_increment_outside_the_unit_ball(emu_pass, monkeypatch):
    import test_gpu_g2o_graphs as T
    T.test_rotation_increment_outside_the_unit_ball(monkeypatch)


@pytest.mark.parametrize("near_ey", [False, True])
def test_makerot0_degenerate_normals(emu_pass, near_ey):
    import test_gpu_g2o_graphs as T
    T.test_makerot0_degenerate_normals(near_ey, n_views=3, n_points=600)


@pytest.mark.parametrize("recomputed", [False, True])
def test_lm_and_g2o_interleaved(emu_pass, oracle, recomputed):
    import test_gpu_g2o_graphs as T
    T.test_lm_and_g2o_interleaved_on_one_engine(oracle, recomputed)
