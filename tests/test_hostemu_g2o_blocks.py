"""The per-edge block check of tests/test_gpu_g2o_blocks.py on the miniature CUDA model in tools/hostemu, with the threads of a
CTA in ascending and in random order: every storage mode at the 1024-slot tile with both costs and every eps, and the readout's
state rules, the build chi2 after a failed factorisation and the component solve.  The hardware's roundings (FMA contraction)
are covered by `pytest -m gpu`."""
import pytest

from test_hostemu_components import emu  # noqa: F401  (the module-scoped host-model fixture, both thread orders)


@pytest.mark.parametrize("mode", ["f32", "f32_recomputed_normals", "f64", "f32_no_normals"])
def test_g2o_edge_blocks(emu, mode):  # noqa: F811
    import test_gpu_g2o_blocks as B
    if emu.order != "ascending" and mode not in ("f32", "f64"):
        pytest.skip("second pass: the two point storages")
    B.run_g2o_block_cases(1024, mode, sets=None if emu.order == "ascending" else ("rigid", "nonrigid"))


def test_g2o_readout_state(emu):  # noqa: F811
    import test_gpu_g2o_blocks as B
    B.check_readout_state_and_interleaving()
    B.check_failed_factorisation_build_chi2()
    B.check_components()
