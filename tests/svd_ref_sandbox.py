"""
The reference's own ``sklearn/svd.py`` (``BiasedSVDScorer`` over scikit-learn's ``TruncatedSVD``) on top of the sandbox
of ``ref_sandbox``, which already loads ``basic/bias.py``, the data classes and ``lenskit.training``; and the recording
of its training on ml-latest-small that ``tests/golden/reference_classes/biased_svd_*.npz`` holds.
"""

from __future__ import annotations

import contextlib
import warnings

import numpy as np

import ref_sandbox

#: what the golden files sample: user rows, item columns, and the users whose ``__call__`` scores are kept
ROWS_U = np.random.default_rng(0).choice(671, 100, replace=False)
ROWS_I = np.random.default_rng(1).choice(9066, 200, replace=False)
SCORE_USERS = np.random.default_rng(2).choice(671, 17, replace=False)
SCORE_ITEMS = np.arange(0, 9066, 29)
UNKNOWN_ID = -12345  # neither a user nor an item id of ml-latest-small
SEED = 42


@contextlib.contextmanager
def svd_modules():
    """``ref_sandbox.reference_modules()`` plus ``lenskit.sklearn.svd``; yields ``{module name: module}``."""
    with ref_sandbox.reference_modules() as mods:
        ref_sandbox._module("lenskit.sklearn", package=True)
        mods["lenskit.sklearn.svd"] = ref_sandbox._load("lenskit.sklearn.svd", "sklearn/svd.py")
        yield mods


def rated_query(ml_small, u: int):
    """The history a rated query carries: user ``u``'s first ten ratings, each raised by one, plus an unknown item."""
    rows = np.flatnonzero(ml_small.users == u)[:10]
    ids = np.append(ml_small.item_ids[ml_small.items[rows]], UNKNOWN_ID)
    ratings = np.append(ml_small.ratings[rows] + 1.0, 3.0).astype(np.float32)
    return ids, ratings


def queries(ml_small):
    """``(user id, history ids or None, history ratings or None)`` of every scored query, in the golden file's order:
    the sampled users, an unknown user, and one user with a rated history."""
    out = [(ml_small.user_ids[u], None, None) for u in SCORE_USERS]
    out.append((UNKNOWN_ID, None, None))
    out.append((ml_small.user_ids[SCORE_USERS[0]], *rated_query(ml_small, int(SCORE_USERS[0]))))
    return out


def score_item_ids(ml_small) -> np.ndarray:
    return np.append(ml_small.item_ids[SCORE_ITEMS], UNKNOWN_ID)


def record(ml_small, k: int, n_iter: int = 5) -> dict:
    """The reference's ``BiasedSVDScorer(embedding_size=k, n_iter=n_iter)`` trained on ml-latest-small under
    ``np.random.seed(SEED)``: biases, singular values, sampled factor rows, ``__call__`` scores and the global
    ``RandomState`` after training."""
    import sklearn

    with svd_modules() as ref, warnings.catch_warnings():
        warnings.simplefilter("ignore")
        svd, items_mod, query_mod = ref["lenskit.sklearn.svd"], ref["lenskit.data._items"], ref["lenskit.data._query"]
        ItemList, RecQuery = items_mod.ItemList, query_mod.RecQuery
        m = svd.BiasedSVDScorer(embedding_size=k, n_iter=n_iter)
        np.random.seed(SEED)
        m.train(ref_sandbox.FakeDataset(ml_small))
        state = np.random.get_state()
        f = m.factorization
        scores = []
        for uid, hist, ratings in queries(ml_small):
            q = RecQuery(user_id=uid, history_items=None if hist is None else ItemList(item_ids=hist, rating=ratings))
            scores.append(np.asarray(m(q, ItemList(item_ids=score_item_ids(ml_small))).scores("numpy"), np.float64))
        return {
            "k": np.int64(k), "n_iter": np.int64(n_iter), "sklearn_version": np.array(sklearn.__version__),
            "global_bias": np.float64(m.bias.global_bias), "item_biases": m.bias.item_biases,
            "user_biases": m.bias.user_biases, "singular_values": f.singular_values_,
            "components": f.components_[:, ROWS_I], "user_components": m.user_components[ROWS_U],
            "scores": np.stack(scores), "state_keys": state[1], "state_pos": np.int64(state[2]),
            "state_gauss": np.array([state[3], state[4]], dtype=np.float64),
        }  # fmt: skip
