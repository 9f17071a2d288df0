"""The cases of tests/test_gpu_seeded_packet.py, small, on the host model of the engine (tools/hostemu): the seeded rounds' packet
fall-through -- votes of settled and unsettled lanes, warp reductions, the lane-register stack, certificates written by the walk --
in ascending and random thread order."""
import pytest

import test_gpu_seeded_packet as T
from test_hostemu_engine import emu  # noqa: F401  (module fixture: the host-model library in place of libmvicp.so)

SMALL = {T.case_settled_and_unsettled_mixed: dict(n=900), T.case_all_settled: dict(n=700), T.case_none_settled: dict(n=900),
         T.case_stale_seeds_and_set_edge: dict(n=700), T.case_ties_and_duplicates: dict(n=6), T.case_partial_warps: {},
         T.case_partial_tiles: dict(ks=(1,)), T.case_georeferenced_fp64: dict(n=600)}


@pytest.mark.parametrize("case", T.CASES, ids=lambda c: c.__name__[5:])
def test_seeded_rounds_on_the_host_model(emu, oracle, case):
    case(oracle, **SMALL[case])


def test_certificates_from_the_packet_walk_on_the_host_model(emu, oracle):
    T.icp_certified(oracle, n_points=1201, warm=4)
