"""The cases of tests/test_gpu_far_packet.py, small, on the host model of the engine (tools/hostemu): the packet walk's votes,
warp reductions and lane-register stack in ascending and random thread order."""
import pytest

import test_gpu_far_packet as T
from test_hostemu_engine import emu  # noqa: F401  (module fixture: the host-model library in place of libmvicp.so)

SMALL = {T.case_unrelated_clouds: dict(n=900), T.case_volume_against_sheet: dict(n=900), T.case_pose_offset_of_many_diameters: dict(n=700),
         T.case_ties_and_duplicates: dict(n=6), T.case_partial_warps: {}, T.case_partial_tiles: dict(ks=(1,)),
         T.case_georeferenced_fp64: dict(n=600)}


@pytest.mark.parametrize("case", T.CASES, ids=lambda c: c.__name__[5:])
def test_far_rounds_on_the_host_model(emu, oracle, case):
    case(oracle, **SMALL[case])
