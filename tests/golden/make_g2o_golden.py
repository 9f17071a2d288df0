"""Writes tests/golden/g2o_trace.npz: the g2o restatement's (tests/g2o_model.py) LM trace on test_g2o_model.golden_problem().
Kept are the trials decided on chi2 differences above 1e-6 relative (the ones that do not hinge on rounding), the final poses
and the number of optimize() calls.  Run from the repository root: python tests/golden/make_g2o_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import g2o_model as G  # noqa: E402
from test_g2o_model import golden_problem  # noqa: E402


def main():
    pts, nor, edges, corr, start = golden_problem()
    prob = G.Problem(pts, nor, edges, corr, [True, False, False], True)
    P, summ, chis, trace = G.optimize(prob, start)
    k = 0
    while k < len(trace) and abs(trace[k, 1] - trace[k, 2]) > 1e-6 * trace[k, 1]:
        k += 1
    np.savez_compressed(os.path.join(HERE, "g2o_trace.npz"), trace=trace[:k], poses=P, calls=summ["calls"], chi=chis)
    print(f"{k} of {len(trace)} trials kept, {summ['calls']} calls, chi2 {chis[0]:.6e} -> {chis[-1]:.6e}")


if __name__ == "__main__":
    main()
