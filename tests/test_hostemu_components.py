"""The per-component LM solve (mvicp_optimize_components, lm_step_components_kernel) compiled against the miniature CUDA model
in tools/hostemu and run through the small cases of tests/test_gpu_components.py on the CPU, with the threads of a CTA in
ascending and in random order.  This checks the logic of the batched state machine, the per-component layouts and the skipping
of finished components; the hardware's roundings are covered by `pytest -m gpu`."""
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
        so2 = str(tmp_path_factory.mktemp("hostemu_cmp") / "libmvicp_hostemu_random.so")
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
    import test_gpu_components as T
    T.check_api(n_points=300)


@pytest.mark.parametrize("name", ["ring_chord", "dst_fixed"])
def test_connected_graph_equals_optimize(emu, oracle, name):
    import test_gpu_components as T
    T.check_connected(oracle, name, params=[T.PARAM_SE3, T.PARAM_QUAT], costs=[T.COST_MIXED], robusts=(True,), n_points=400)


@pytest.mark.parametrize("path", ["unit", "general"])
def test_batch_matches_fresh_engines_and_oracle(emu, oracle, path):
    import test_gpu_components as T
    comps = T.mixed_comps(oracle, n_points=300, nonrigid=path == "general", wide=False)
    T.check_batch(oracle, comps, T.PARAM_SE3, T.COST_P2PLANE, True)


def test_max_iterations_next_to_early_stops(emu, oracle):
    import test_gpu_components as T
    T.check_max_iterations_next_to_early_stops(oracle, n_points=400)


def test_icp_rounds(emu):
    import test_gpu_components as T
    if emu.order != "ascending":
        pytest.skip("slow case: first pass only")
    T.check_icp_rounds(n_pairs=3, n_points=600, rounds=20)
