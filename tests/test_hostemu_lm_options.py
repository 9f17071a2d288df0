"""The LM loop under non-default options and failing steps (tests/test_gpu_lm_options.py), compiled against the miniature CUDA
model in tools/hostemu and run on the CPU with the threads of a CTA in ascending and in random order: every termination, the
zero pivot in the first, a middle and the last block of the shared-memory factor, one mixed-outcome component batch and the
option rules -- small scenes, no 48-view factor.  The hardware's roundings are covered by `pytest -m gpu`."""
import pytest

from test_hostemu_components import emu  # noqa: F401  (the module-scoped host-model fixture, both thread orders)

N = 300
COMBOS = [(0, 0, False), (2, 1, True)]     # (param, cost, robust): angle-axis point-to-point, SE3 point-to-plane robust


@pytest.mark.parametrize("combo", COMBOS, ids=["aa-p2p", "se3-plane-robust"])
@pytest.mark.parametrize("case", ["max_iterations", "gradient", "zero_residual", "min_radius", "reject_then_accept",
                                  "small_radius", "no_scaling", "clamps", "invalid_positions", "model_change"])
def test_joint_cases(emu, oracle, case, combo):  # noqa: F811
    import test_gpu_lm_options as L
    if emu.order != "ascending" and combo != COMBOS[1]:
        pytest.skip("second pass: one parameterisation")
    getattr(L, "check_" + case)(oracle, N, *combo)


@pytest.mark.parametrize("mode,path,param", [("f32", "unit", 0), ("f64", "general", 2)])
def test_storage_failures(emu, oracle, mode, path, param):  # noqa: F811
    import test_gpu_lm_options as L
    L.check_storage_failures(oracle, mode, path, param, N)


def test_mixed_outcome_batch(emu, oracle):  # noqa: F811
    import test_gpu_lm_options as L
    L.check_mixed_batch(oracle, N, 2, 1, True, wide=False)


def test_option_rules(emu):  # noqa: F811
    import test_gpu_lm_options as L
    L.check_option_rules(200)
