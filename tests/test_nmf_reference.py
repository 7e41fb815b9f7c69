"""
NMF against the reference's own ``NMFScorer`` without a GPU: the host restatement of the descent (tests/nmf_oracle.py,
with the f64 Gram), from scikit-learn's initialisation under ``np.random.seed``, against the recordings of the
reference class on ml-latest-small.  CPU only.

The reference's side comes from a lenskit/lkpy checkout when there is one, else from
``tests/golden/reference_classes/nmf_k*.npz``, which ``LK_RECORD_REFERENCE_GOLDEN=1`` rewrites from the checkout
(tests/nmf_ref_sandbox.py).
"""

import os
from pathlib import Path

import numpy as np
import pytest

import nmf_oracle as no
import nmf_ref_sandbox as nrs
import ref_sandbox

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden" / "reference_classes"
RECORD = os.environ.get("LK_RECORD_REFERENCE_GOLDEN") == "1"
GOLDEN_K = (16, 64)

# Relative Frobenius bounds against the recordings, for factors sampled rows and for the scores of the sampled users.
# Measured for the host restatement (scikit-learn's own initialisation, f64 Grams), the recording's 120 and 178
# iterations reproduced exactly:
#   k = 16: W 5.6e-5, H 3.5e-5, scores 2.6e-6        k = 64: W 3.0e-5, H 1.2e-5, scores 1.2e-6
# and for the device NMFScorer (cuSOLVER's SVD in the initialisation as well), tests/test_nmf_reference_gpu.py:
#   k = 16: W 1.7e-4, H 1.8e-4, scores 1.2e-4        k = 64: W 4.6e-4, H 2.7e-4, scores 5.9e-5
# The bounds leave a factor of about three over the larger of each pair.
FACTOR_TOL = {16: 6e-4, 64: 1.5e-3}
SCORE_TOL = {16: 4e-4, 64: 2e-4}


def reference_golden(ml_small, k: int) -> dict:
    """The reference's values for ``embedding_size=k``: recorded live when asked to, else read from the golden file."""
    path = GOLD / f"nmf_k{k}.npz"
    if RECORD:
        assert ref_sandbox.available(), "recording needs the reference checkout"
        np.savez_compressed(path, **nrs.record(ml_small, k))
    with np.load(path) as z:
        return {name: z[name] for name in z.files}


def rel(a, b) -> float:
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def check_state(g: dict) -> None:
    """The global ``RandomState`` is where the reference's training left it."""
    state = np.random.get_state()
    assert np.array_equal(state[1], g["state_keys"]) and state[2] == g["state_pos"]
    assert np.array_equal([state[3], state[4]], g["state_gauss"])


def check_scores(g: dict, user_components, item_components, k: int) -> float:
    """``W[u] · H[:, i]`` of the sampled users against the recorded ``__call__`` scores; the unknown item, the unknown
    user and the unknown user with a history score NaN there.  Returns the relative difference."""
    scores = g["scores"]
    assert np.isnan(scores[-2:]).all() and np.isnan(scores[:-2, -1]).all()
    ours = item_components[nrs.SCORE_ITEMS].astype(np.float64) @ user_components[nrs.SCORE_USERS].T.astype(np.float64)
    err = rel(ours.T, scores[:-2, :-1])
    assert err < SCORE_TOL[k]
    return err


@pytest.mark.parametrize("k", GOLDEN_K)
def test_host_loop_is_the_reference(ml_small, k):
    """scikit-learn's initialisation and the restated loop under ``np.random.seed(SEED)`` reproduce the recording's
    iteration count and global state exactly, and its factors and scores to rounding."""
    pytest.importorskip("sklearn")
    from sklearn.decomposition._nmf import _initialize_nmf

    g = reference_golden(ml_small, k)
    X = nrs.indicator(ml_small)
    np.random.seed(nrs.SEED)
    W0, H0 = _initialize_nmf(X, k)
    check_state(g)
    W, H, n_iter = no.fit(X, W0, H0, max_iter=200)
    assert n_iter == g["n_iter"]
    assert rel(W[nrs.ROWS_U], g["user_components"]) < FACTOR_TOL[k]
    assert rel(H.T[nrs.ROWS_I], g["item_components"]) < FACTOR_TOL[k]
    check_scores(g, W, np.ascontiguousarray(H.T), k)
