"""The per-edge block check of tests/test_gpu_lm_blocks.py on the miniature CUDA model in tools/hostemu, with the threads of a
CTA in ascending and in random order: every storage mode at the 1024-slot tile, every parameterisation on the unit and the
general path, the three costs, and the loss off, at the edges' weights and at a tiny and a huge weight.  The hardware's
roundings (FMA contraction, rsqrt) are covered by `pytest -m gpu`."""
import pytest

from test_hostemu_components import emu  # noqa: F401  (the module-scoped host-model fixture, both thread orders)


@pytest.mark.parametrize("mode", ["f32", "f32_recomputed_normals", "f64", "f32_no_normals"])
def test_edge_blocks(emu, oracle, mode):  # noqa: F811
    import test_gpu_lm_blocks as B
    if emu.order != "ascending" and mode not in ("f32", "f64"):
        pytest.skip("second pass: the two point storages")
    B.run_block_cases(oracle, 1024, mode, use_oracle=mode == "f64")


def test_readout_state(emu, oracle):  # noqa: F811
    import test_gpu_lm_blocks as B
    B.test_readout_state_and_last_evaluation(oracle)
    B.test_readout_component_without_free_frame(oracle)
