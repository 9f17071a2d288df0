"""The seeded rounds' packet search (csrc/knn.cuh: nn_search_packet, nn_packet_walk) compiled by g++ against the host CUDA model
(tools/hostemu) and run one warp at a time against a brute force (tools/knn_packet_host_check.cpp): exact index and d^2 with and
without the neighbour lists, and every certificate margin written by the walk at most the true gap to the runner-up.  Warps mix
settled and walking lanes, seed kinds and query kinds; the last warp is partial.  Lanes run in ascending and in random order."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("knnpacket") / "knn_packet_host_check")
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    r = subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-w", "-I" + os.path.join(ROOT, "tools", "hostemu"), "-I" + cuda_inc,
                        "-o", exe, os.path.join(ROOT, "tools", "knn_packet_host_check.cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.parametrize("order", ["ascending", "random"])
@pytest.mark.parametrize("mode", [0, 1], ids=["fp32-storage", "fp64-storage"])
@pytest.mark.parametrize("n", [1, 9, 1000, 12345])
def test_packet_search_and_its_certificates_on_host(harness, n, mode, order):
    env = dict(os.environ, HOSTEMU_ORDER=order)
    r = subprocess.run([harness, str(n), "24", str(31 + n), str(mode)], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-2000:]
    assert " 0 mismatches" in r.stdout
