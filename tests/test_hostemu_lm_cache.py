"""tests/test_gpu_lm_cache.py (optimize, optimize_components, optimize_g2o, optimize with another fixed set, optimize_components
on one engine, each against a fresh engine) compiled against the miniature CUDA model in tools/hostemu and run at small sizes on
the CPU, with the threads of a CTA in ascending and in random order."""
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
        so2 = str(tmp_path_factory.mktemp("hostemu_cache") / "libmvicp_hostemu_random.so")
        shutil.copy(so, so2); so = so2
        os.environ["HOSTEMU_ORDER"] = "random"
    lib = C.CDLL(so); lib.mvicp_last_error.restype = C.c_char_p
    os.environ.pop("HOSTEMU_ORDER", None)
    lib.order = request.param
    saved = _lib._lib
    _lib._lib = lib
    yield lib
    _lib._lib = saved


@pytest.mark.parametrize("mode", ["f32", "f32_recomputed_normals", "f64", "f32_no_normals"])
def test_sequence_matches_fresh_engines(emu, oracle, mode):
    import test_gpu_lm_cache as L
    if emu.order != "ascending" and mode != "f32":
        pytest.skip("one storage mode in the random pass")
    L.check_sequence(oracle, L.cache_comps(oracle, n_points=200, mode=mode), mode, max_iter=4, g2o_calls=2)
