"""The step check of tests/test_gpu_lm_step.py on the miniature CUDA model in tools/hostemu, with the threads of a CTA in
ascending and in random order: every parameterisation and path, the envelope shapes of up to 10 views, every trust-region
setting, a rejected step followed by an accepted one, a component batch without the wide component, the ill-conditioned
patch and the clouds far from the origin.  The hardware's roundings (FMA contraction, rsqrt) and the wide graphs are
covered by `pytest -m gpu`."""
import pytest

from test_hostemu_components import emu  # noqa: F401  (the module-scoped host-model fixture, both thread orders)

SMALL_SHAPES = ["ring_chord", "dst_only", "dst_fixed", "two_components", "chain", "star", "single"]


@pytest.mark.parametrize("name", ["aa", "quat", "se3", "quat-general", "se3-general", "quat-mixed", "aa-p2p"])
def test_step_parameterisations_and_paths(emu, oracle, name):  # noqa: F811
    import test_gpu_lm_step as S
    S.check_param(oracle, name)


@pytest.mark.parametrize("name", SMALL_SHAPES)
def test_step_envelope_shapes(emu, oracle, name):  # noqa: F811
    import test_gpu_lm_step as S
    S.check_shape(oracle, name)


@pytest.mark.parametrize("name", ["defaults", "gauss_newton", "tiny_radius", "no_scaling", "min_diag_binds", "max_diag_binds",
                                  "min_diag_zero"])
def test_step_trust_region_settings(emu, oracle, name):  # noqa: F811
    import test_gpu_lm_step as S
    S.check_trust(oracle, name)


def test_step_rejected_then_accepted(emu, oracle):  # noqa: F811
    import test_gpu_lm_step as S
    S.check_reject_then_accept(oracle)


def test_step_component_batch(emu, oracle):  # noqa: F811
    import test_gpu_lm_step as S
    S.check_components(oracle, n_points=400, wide=False)


def test_step_ill_conditioned(emu, oracle):  # noqa: F811
    import test_gpu_lm_step as S
    S.check_ill_conditioned(oracle)


@pytest.mark.parametrize("param", [0, 1])
def test_step_far_from_origin(emu, oracle, param):  # noqa: F811
    import test_gpu_lm_step as S
    S.check_far(oracle, param)
