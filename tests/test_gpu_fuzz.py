"""Adversarial clouds on the GPU: the device-built search structure (tree_gpu.cuh) and the hardware fp32 screen (sqrt.approx
bounds in knn.cuh) against the oracle, an independent numpy brute force and the host-built tree (MVICP_FLAG_HOST_BUILD), on the
seeded fuzz corpus of tools/fuzz_hostemu.py (collinear / identical / quantised clouds, tiny clouds, scales 1e-3..1e3, offsets,
georeferenced scans at 1e5-1e6 m), the converged-round shortcuts, the LM step, degenerate clouds around the leaf and level
boundaries, and the k-NN lists and normals at every k the ABI accepts.  The k-NN and normals tests also run on the host model
of the engine (tests/test_hostemu_engine.py)."""
import functools
import os
import sys

import numpy as np
import pytest

from mv_lm_icp_b200 import Engine, _lib
from mv_lm_icp_b200._lib import MvicpError
from mv_lm_icp_b200.api import FLAG_HOST_BUILD, FLAG_NO_ADJ, FLAG_NO_OBB, FLAG_STEP_LOOP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MVICP_ERR_INVALID = 1

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fuzz(oracle):
    """The case functions of tools/fuzz_hostemu.py, run on the product library."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import fuzz_hostemu
    assert _lib.lib()._name == _lib.LIB_PATH
    return fuzz_hostemu


def _same_nn(a, b):
    return len(a) == len(b) and all(np.array_equal(i0, i1) and np.array_equal(d0.view(np.uint64), d1.view(np.uint64))
                                    for r0, r1 in zip(a, b) for (i0, d0), (i1, d1) in zip(r0, r1))


def _device_and_host_tree(fuzz, case):
    """The case's rounds on a device-built and on a host-built tree (every round against the oracle, the first against the brute
    force): the two must agree bit for bit."""
    dev = fuzz.run_case(dict(case, flags=case["flags"] & ~FLAG_HOST_BUILD), brute=True)
    host = fuzz.run_case(dict(case, flags=case["flags"] | FLAG_HOST_BUILD))
    assert _same_nn(dev, host), (case["name"], "device tree vs host tree")


@pytest.mark.parametrize("seed", range(200))
def test_cold_and_seeded_rounds(fuzz, seed):
    _device_and_host_tree(fuzz, fuzz.one_case(seed))


@pytest.mark.parametrize("seed", range(64))
def test_georeferenced_rounds(fuzz, seed):
    _device_and_host_tree(fuzz, fuzz.geo_case(seed))


def test_converged_rounds(fuzz):
    """Certified matches and the guessed median select against an engine without either (FLAG_NO_CERT | FLAG_NO_SELECT_GUESS),
    bit for bit, over 100 seeds; the shortcuts must actually have been taken, or the comparison proves nothing."""
    guess = cert = reused = 0
    for seed in range(100):
        _, _, g, c, r = fuzz.one_steady(seed)
        guess += g; cert += c; reused += r
    print(f"converged rounds, 100 seeds: select_guess_rounds {guess}, cert_rounds {cert}, cert_reused {reused}")
    assert guess > 0 and cert > 0 and reused > 0


@pytest.mark.parametrize("seed", range(40))
def test_lm_step(fuzz, seed):
    fuzz.one_lm(seed)


# ---- degenerate clouds: the device tree around the leaf (8) and level boundaries ------------------------------------------------
DEGENERATE_SIZES = (9, 16, 17, 64, 65, 513, 4097)
DEGENERATE_SHAPES = ("identical", "collinear", "sheet", "tilted sheet", "grid", "offset 1e5")


def _degenerate(shape, n, rng):
    """(cloud, spread): the spread sets the scale of the query noise."""
    u, v = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    if shape == "identical":
        return np.tile(rng.normal(size=3), (n, 1)), 1.0
    if shape == "collinear":
        return np.outer(u, [1.0, 0.5, -0.25]) + rng.normal(size=3), 1.0
    if shape == "sheet":        # z constant
        return np.stack([u, v, np.full(n, 0.3)], 1), 1.0
    if shape == "tilted sheet":
        w = np.array([0.3, -0.5, 0.8]); w /= np.linalg.norm(w)
        a = np.cross(w, [1.0, 0, 0]); a /= np.linalg.norm(a); b = np.cross(w, a)
        return np.outer(u, a) + np.outer(v, b), 1.0
    if shape == "grid":         # coarse lattice: duplicates, and queries equidistant from several points
        return np.round(rng.uniform(-1, 1, (n, 3)) * 3) / 4, 1.0
    return rng.normal(size=(n, 3)) * 0.01 + np.array([1e5, -1e5, 1e5]), 0.01    # fp32 spacing 0.0078 at 1e5


@functools.lru_cache(maxsize=2)
def _degenerate_set(fp64):
    """Every (shape, size) cloud and a query cloud near it: noisy copies of its points, midpoints of pairs of its points
    (equidistant from both), points spread over its bounding box.  fp32 storage: every coordinate fp32-exact; fp64: none."""
    rng = np.random.default_rng(41 + fp64)
    clouds, queries, names = [], [], []
    for shape in DEGENERATE_SHAPES:
        for n in DEGENERATE_SIZES:
            c, spread = _degenerate(shape, n, rng)
            q = np.concatenate([c + rng.normal(0, 1e-3 * spread, c.shape), 0.5 * (c + c[rng.permutation(n)]),
                                c.min(0) - 0.1 * spread + (np.ptp(c, 0) + 0.2 * spread) * rng.uniform(size=(n // 4 + 1, 3))])
            if fp64 and shape == "grid":
                c = c + 0.1                                                 # off the fp32 grid (the other shapes are already)
            elif not fp64:
                c = c.astype(np.float32).astype(np.float64); q = q.astype(np.float32).astype(np.float64)
            clouds.append(c); queries.append(q); names.append((shape, n))
    return clouds, queries, names


def _lowest_equal_index(c):
    """For every point, the lowest index of a point with the same coordinates."""
    _, first, inv = np.unique(c, axis=0, return_index=True, return_inverse=True)
    return first[inv.reshape(-1)].astype(np.int32)


@pytest.mark.parametrize("fp64", [False, True], ids=["fp32-storage", "fp64-storage"])
def test_device_tree_on_degenerate_clouds(fuzz, oracle, fp64):
    """Every cloud against itself: each point's match is the lowest index among the points equal to it, at d2 = 0.  Query clouds
    against the brute force, cold and seeded (the query frame moved by a small translation), under every search schedule and
    on the host-built tree."""
    brute_nn = fuzz.brute_nn
    clouds, queries, names = _degenerate_set(fp64)
    assert all(np.array_equal(c.astype(np.float32).astype(np.float64), c) for c in clouds) != fp64
    M = len(clouds)
    frames = clouds + clouds + queries
    edges = [(M + i, i) for i in range(M)] + [(2 * M + i, i) for i in range(M)]
    rounds = []
    for shift in (0.0, 3e-4):
        P = [np.eye(4) for _ in frames]
        for i in range(M):
            P[2 * M + i][:3, 3] = shift * (0.01 if names[i][0] == "offset 1e5" else 1.0)
        rounds.append((P, [brute_nn(clouds[i], oracle.edge_queries(queries[i], P[2 * M + i], P[i])) for i in range(M)]))
    self_ref = [_lowest_equal_index(c) for c in clouds]
    for flags in (0, FLAG_NO_OBB, FLAG_NO_ADJ, FLAG_STEP_LOOP, FLAG_HOST_BUILD):
        eng = Engine(flags=flags); eng.set_frames(frames, None); eng.set_graph(edges)
        for rnd, (P, ref) in enumerate(rounds):
            eng.set_poses(P, [1] + [0] * (len(frames) - 1)); eng.correspond(0.05)
            for i in range(M):
                idx, d2 = eng.get_nn(i)
                assert np.all(d2 == 0.0) and np.array_equal(idx, self_ref[i]), (flags, rnd, names[i], "self")
                idx, d2 = eng.get_nn(M + i)
                bi, bd = ref[i]
                assert np.array_equal(d2.view(np.uint64), bd.view(np.uint64)), (flags, rnd, names[i], "d2", int(np.sum(d2 != bd)))
                assert np.array_equal(idx, bi), (flags, rnd, names[i], "idx", int(np.sum(idx != bi)))
        eng.close()


# ---- k-NN lists and normals at every k --------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=1)
def _knn_clouds():
    rng = np.random.default_rng(23)
    x, y = rng.uniform(-1, 1, 1500), rng.uniform(-1, 1, 1500)
    base = rng.normal(size=(200, 3)).astype(np.float32).astype(np.float64)
    return {
        "jittered surface": np.stack([x, y, 0.2 * np.sin(3 * x) * np.cos(2 * y) + 1e-3 * rng.normal(size=1500)], 1),
        "flat sheet": np.stack([rng.uniform(-1, 1, 1200), rng.uniform(-1, 1, 1200), np.zeros(1200)], 1).astype(np.float32).astype(np.float64),
        "quantised grid": np.round(rng.uniform(-1, 1, (1200, 3)) * 4) / 4,              # ties at the k-th distance
        "triplicated": np.concatenate([base, base, base])[rng.permutation(600)],
        "5 points": rng.normal(size=(5, 3)),                                               # n < k: -1 padded tail
        "1003 points": rng.normal(size=(1003, 3)).astype(np.float32).astype(np.float64),   # partial last leaf
        "fp64, offset": rng.normal(size=(1500, 3)) * 0.1 + np.array([1e4, -2e4, 3e4]),
    }


def brute_knn(c, k):
    """The k nearest points of every point (itself included), ordered by (d2, index), d2 = (d0*d0 + d1*d1) + d2*d2 in fp64;
    -1 where the cloud has fewer than k points."""
    n = len(c); out = np.full((n, k), -1, np.int32)
    ar = np.arange(n)
    for a in range(n):
        d = c[a] - c
        D = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        o = np.lexsort((ar, D))[:k]
        out[a, :len(o)] = o
    return out


@functools.lru_cache(maxsize=8)
def _brute16(name):
    return brute_knn(_knn_clouds()[name], 16)


def test_knn_self_every_k():
    """mvicp_knn_self for k = 1..16 against the brute force; the neighbour-list shortcut (k <= 8: the list is full after the
    point's own leaf) and the host-built tree must give identical lists; k = 0 and 17 are rejected."""
    for name, c in _knn_clouds().items():
        ref = _brute16(name)
        for flags in (0, FLAG_NO_ADJ, FLAG_HOST_BUILD):
            eng = Engine(flags=flags); eng.set_frames([c], None)
            for k in range(1, 17):
                nn = eng.knn_self(0, k)
                assert np.array_equal(nn, ref[:, :k]), (name, flags, k, int(np.sum(np.any(nn != ref[:, :k], 1))))
            for k in (0, 17):
                with pytest.raises(MvicpError) as e:
                    eng.knn_self(0, k)
                assert e.value.code == MVICP_ERR_INVALID
            eng.close()


def test_normals_every_k():
    """mvicp_recompute_normals for k = 3..16 against numpy.linalg.eigh of the brute-force neighbourhoods: within 1e-9 (up to
    sign) wherever the eigen-gap (w1 - w0) / w2 exceeds 1e-3; on every point, degenerate neighbourhoods included: finite, unit
    norm, n.z <= 0.  k = 2 and 17 are rejected."""
    for name, c in _knn_clouds().items():
        ref16 = _brute16(name)
        eng = Engine(); eng.set_frames([c], None)
        checked = 0
        for k in range(3, 17):
            nor = eng.recompute_normals(k)[0][0]
            assert np.all(np.isfinite(nor)) and np.all(nor[:, 2] <= 0), (name, k)
            assert np.max(np.abs(np.linalg.norm(nor, axis=1) - 1)) < 1e-12, (name, k)
            nb = ref16[:, :min(k, len(c))]
            P = c[nb]; D = P - P.mean(1, keepdims=True)
            w, V = np.linalg.eigh(np.einsum("nki,nkj->nij", D, D))
            sep = (w[:, 1] - w[:, 0]) > 1e-3 * w[:, 2]
            v = V[:, :, 0]
            err = np.minimum(np.abs(nor - v).max(1), np.abs(nor + v).max(1))
            assert np.all(err[sep] < 1e-9), (name, k, float(err[sep].max()))
            checked += int(sep.sum())
        if name not in ("triplicated", "5 points"):
            assert checked > len(c), name          # most neighbourhoods are well separated: the comparison is not vacuous
        for k in (2, 17):
            with pytest.raises(MvicpError) as e:
                eng.recompute_normals(k)
            assert e.value.code == MVICP_ERR_INVALID
        eng.close()
