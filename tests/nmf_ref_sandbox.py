"""
The reference's own ``sklearn/nmf.py`` (``NMFScorer`` over scikit-learn's ``non_negative_factorization``) on top of the
sandbox of ``ref_sandbox``, which already loads the data classes, ``lenskit.config.common`` and ``lenskit.training``;
and the recording of its training on ml-latest-small that ``tests/golden/reference_classes/nmf_k*.npz`` holds.
"""

from __future__ import annotations

import contextlib
import warnings

import numpy as np

import ref_sandbox
from svd_ref_sandbox import ROWS_I, ROWS_U, SCORE_ITEMS, SCORE_USERS, SEED, UNKNOWN_ID  # noqa: F401


@contextlib.contextmanager
def nmf_modules():
    """``ref_sandbox.reference_modules()`` plus ``lenskit.sklearn.nmf``; yields ``{module name: module}``."""
    with ref_sandbox.reference_modules() as mods:
        ref_sandbox._module("lenskit.sklearn", package=True)
        mods["lenskit.sklearn.nmf"] = ref_sandbox._load("lenskit.sklearn.nmf", "sklearn/nmf.py")
        yield mods


def queries(ml_small):
    """``(user id, history ids or None)`` of every scored query, in the golden file's order: the sampled users, an
    unknown user, and an unknown user with a history (NaN as well: NMF scores only known users)."""
    out = [(ml_small.user_ids[u], None) for u in SCORE_USERS]
    out.append((UNKNOWN_ID, None))
    out.append((UNKNOWN_ID, ml_small.item_ids[ml_small.items[ml_small.users == SCORE_USERS[0]][:10]]))
    return out


def score_item_ids(ml_small) -> np.ndarray:
    """The scored items: every 29th item, then an unknown one."""
    return np.append(ml_small.item_ids[SCORE_ITEMS], UNKNOWN_ID)


def indicator(ml_small):
    """The reference's training matrix: ``interactions().matrix().scipy(layout="csr")``, f32 ones."""
    return ref_sandbox._MatrixView(ml_small).scipy(None, layout="csr")


def record(ml_small, k: int) -> dict:
    """The reference's ``NMFScorer(embedding_size=k)`` trained on ml-latest-small under ``np.random.seed(SEED)``:
    the iteration count (from ``non_negative_factorization`` under the same seed, since the scorer discards it),
    sampled factor rows, ``__call__`` scores and the global ``RandomState`` after training."""
    import sklearn
    from sklearn.decomposition import non_negative_factorization

    with nmf_modules() as ref, warnings.catch_warnings():
        warnings.simplefilter("ignore")
        nmf, items_mod, query_mod = ref["lenskit.sklearn.nmf"], ref["lenskit.data._items"], ref["lenskit.data._query"]
        ItemList, RecQuery = items_mod.ItemList, query_mod.RecQuery
        m = nmf.NMFScorer(embedding_size=k)
        np.random.seed(SEED)
        m.train(ref_sandbox.FakeDataset(ml_small))
        state = np.random.get_state()
        np.random.seed(SEED)
        _W, _H, n_iter = non_negative_factorization(indicator(ml_small), n_components=k)
        scores = []
        for uid, hist in queries(ml_small):
            q = RecQuery(user_id=uid, history_items=None if hist is None else ItemList(item_ids=hist))
            scores.append(np.asarray(m(q, ItemList(item_ids=score_item_ids(ml_small))).scores("numpy"), np.float64))
        return {
            "k": np.int64(k), "n_iter": np.int64(n_iter), "sklearn_version": np.array(sklearn.__version__),
            "user_components": m.user_components[ROWS_U], "item_components": m.item_components[ROWS_I],
            "scores": np.stack(scores), "state_keys": state[1], "state_pos": np.int64(state[2]),
            "state_gauss": np.array([state[3], state[4]], dtype=np.float64),
        }  # fmt: skip
