"""
The device ``NMFScorer`` against the recordings of the reference's own ``NMFScorer`` on ml-latest-small
(tests/golden/reference_classes/nmf_k*.npz, tests/nmf_ref_sandbox.py): ``train`` under ``np.random.seed`` gives the
reference's iteration count and leaves the global ``RandomState`` where the reference left it; ``user_components``,
``item_components`` and the ``__call__`` scores (NaN for an unknown item, an unknown user, and an unknown user with a
history) agree to the measured tolerances.
"""

import numpy as np
import pytest

import nmf_ref_sandbox as nrs
import test_nmf_reference as host
from lkpy_b200.components import Dataset, ItemList, RecQuery
from lkpy_b200.nmf import NMFScorer

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("k", host.GOLDEN_K)
def test_scorer_is_the_reference(ml_small, k):
    g = host.reference_golden(ml_small, k)
    m = NMFScorer(embedding_size=k)
    np.random.seed(nrs.SEED)
    m.train(Dataset(ml_small))
    host.check_state(g)
    assert m.n_iter_ == g["n_iter"]
    assert m.user_components.dtype == m.item_components.dtype == np.float32
    assert m.user_components.shape == (ml_small.n_users, k) and m.item_components.shape == (ml_small.n_items, k)
    errs = (host.rel(m.user_components[nrs.ROWS_U], g["user_components"]),
            host.rel(m.item_components[nrs.ROWS_I], g["item_components"]))  # fmt: skip
    scores = []
    for uid, hist in nrs.queries(ml_small):
        q = RecQuery(uid, None if hist is None else ItemList(item_ids=hist))
        scores.append(m(q, ItemList(item_ids=nrs.score_item_ids(ml_small))).scores())
    scores = np.stack(scores)
    assert np.array_equal(np.isnan(scores), np.isnan(g["scores"]))
    score_err = host.rel(scores[:-2, :-1], g["scores"][:-2, :-1])
    print(f"k={k}: n_iter {m.n_iter_}; user components {errs[0]:.2e}, item components {errs[1]:.2e}, "
          f"scores {score_err:.2e}")  # fmt: skip
    assert errs[0] < host.FACTOR_TOL[k] and errs[1] < host.FACTOR_TOL[k]
    assert score_err < host.SCORE_TOL[k]
    assert host.check_scores(g, m.user_components, m.item_components, k) < host.SCORE_TOL[k]
