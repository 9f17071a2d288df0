"""Pin of the oracle's restated cost functors against the REFERENCE's own functor text (round-1 verdict, item 8).

oracle/_ref/libref_functors.so is include/icp-ceres.h (all twelve functors) + include/eigen_quaternion.h compiled UNMODIFIED from
/root/reference against oracle/stubs/ (mini Eigen interface, Ceres class shells, three members of Sophus::SE3Group) and
differentiated with the oracle's Jet (oracle/ref_functors.cpp; recipe oracle/Makefile).  It is built only where the reference
tree is present; elsewhere the tests compare with its outputs on the first inputs of every case (tests/golden/functor_pin.npz).

Tolerance: the restatement and the reference text may associate 3-term sums differently (Eigen 3.3 reduces x0 + (x1 + x2),
the restatement folds left), so values are compared to a few ulps of the magnitudes that enter them, not bit for bit."""
import numpy as np
import pytest

EPS = np.finfo(np.float64).eps


def _rand_pose(rng, param, unit=True):
    if param == 0:
        return np.concatenate([rng.normal(0, 0.8, 3), rng.normal(0, 0.5, 3)])
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    if not unit:
        q *= rng.uniform(0.98, 1.02)       # the reference runs its functors on non-unit quaternions too (non-rigid sample poses)
    return np.concatenate([q, rng.normal(0, 0.5, 3)])


def _global_cases(param, plane):
    rng = np.random.default_rng(100 + 10 * param + plane)
    for it in range(10_000 // 6 + 1):
        c1 = _rand_pose(rng, param, unit=it % 3 != 0); c2 = _rand_pose(rng, param, unit=it % 3 != 0)
        if param == 0 and it % 50 == 0:
            c1[:3] = rng.normal(0, 1e-9, 3)     # first-order branch of AngleAxisRotatePoint (theta^2 <= DBL_EPSILON)
        src = rng.normal(0, 0.3, 3); dst = rng.normal(0, 0.3, 3); nor = rng.normal(size=3); nor /= np.linalg.norm(nor)
        yield c1, c2, src, dst, nor


def _pairwise_cases(param, plane):
    rng = np.random.default_rng(200 + 10 * param + plane)
    for it in range(1000):
        c1 = _rand_pose(rng, param)
        src = rng.normal(0, 0.3, 3); dst = rng.normal(0, 0.3, 3); nor = rng.normal(size=3); nor /= np.linalg.norm(nor)
        yield c1, src, dst, nor


def _quat_cases():
    rng = np.random.default_rng(7)
    for it in range(2000):
        x = rng.normal(size=4); x /= np.linalg.norm(x)
        d = rng.normal(0, 0.3, 3) if it % 10 else np.zeros(3)
        yield x, d


class _Reference:
    """The reference's functor text: the library itself when oracle/_ref was built, otherwise its outputs on the first inputs
    of every case, stored in tests/golden/functor_pin.npz (make_golden.py:functor_pin)."""

    def __init__(self, O, golden):
        self.O, self.g, self.lib = O, golden, O.ref_functors()

    def has(self, key, it):
        return self.lib is not None or it < len(self.g[key + "_r"])

    def global_(self, key, it, param, plane, *args):
        if self.lib is not None:
            return self.O.functor_eval(param, plane, *args, "ref")
        return self.g[key + "_r"][it], self.g[key + "_j"][it]

    def pairwise(self, key, it, param, plane, *args):
        if self.lib is not None:
            return self.O.functor_eval_pairwise_ref(param, plane, *args)
        return self.g[key + "_r"][it], self.g[key + "_j"][it]

    def quat(self, it, x, d):
        if self.lib is None:
            return self.g["quat_r"][it], self.g["quat_j"][it]
        import ctypes as C
        P = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
        out = np.zeros(4); self.lib.ref_quat_plus(P(x), P(d), P(out))
        j = np.zeros(12); self.lib.ref_quat_jacobian(P(x), P(j))
        return out, j


@pytest.fixture(scope="module")
def R(oracle, golden_dir):
    return _Reference(oracle, np.load(f"{golden_dir}/functor_pin.npz"))


@pytest.mark.parametrize("param", [0, 1, 2])
@pytest.mark.parametrize("plane", [0, 1])
def test_global_functors_match_reference_text(R, param, plane):
    key = f"global_{param}{plane}"
    worst_r = worst_j = 0.0
    for it, (c1, c2, src, dst, nor) in enumerate(_global_cases(param, plane)):
        if not R.has(key, it):
            break
        r0, j0 = R.O.functor_eval(param, plane, c1, c2, src, dst, nor, "oracle")
        r1, j1 = R.global_(key, it, param, plane, c1, c2, src, dst, nor)
        scale = 1.0 + np.abs(c1).max() + np.abs(c2).max() + np.abs(src).max() + np.abs(dst).max()
        worst_r = max(worst_r, np.abs(r0 - r1).max() / scale); worst_j = max(worst_j, np.abs(j0 - j1).max() / scale)
    assert worst_r <= 16 * EPS and worst_j <= 32 * EPS, (worst_r / EPS, worst_j / EPS)


@pytest.mark.parametrize("param", [0, 1, 2])
@pytest.mark.parametrize("plane", [0, 1])
def test_pairwise_functors_are_the_global_ones_with_identity_dst(R, param, plane):
    """icp-ceres.h:320-552 (one pose) against the restated global functor with an identity dst pose -- the way the engine and the
    oracle run the pairwise solvers (a two-frame problem whose frame 0 is constant at identity)."""
    key = f"pairwise_{param}{plane}"
    ident = np.zeros(6) if param == 0 else np.array([0, 0, 0, 1.0, 0, 0, 0])
    G = 6 if param == 0 else 7
    for it, (c1, src, dst, nor) in enumerate(_pairwise_cases(param, plane)):
        if not R.has(key, it):
            break
        r0, j0 = R.O.functor_eval(param, plane, c1, ident, src, dst, nor, "oracle")
        r1, j1 = R.pairwise(key, it, param, plane, c1, src, dst, nor)
        assert np.abs(r0 - r1).max() <= 32 * EPS and np.abs(j0[:, :G] - j1).max() <= 64 * EPS


def test_quaternion_parameterisation_matches_reference_text(R):
    """eigen_quaternion.h:89-117: Plus (left-multiplied [sin|d| d/|d|, cos|d|], identity at d = 0) and the hand-written 4x3 Jacobian."""
    import ctypes as C
    P = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    for it, (x, d) in enumerate(_quat_cases()):
        if not R.has("quat", it):
            break
        out, j = R.quat(it, x, d)
        assert np.abs(out - R.O.quat_plus(x, d)).max() <= 8 * EPS
        j0 = np.zeros(12); R.O.lib().orc_quat_jacobian(P(x), P(j0))
        assert np.array_equal(j, j0)
