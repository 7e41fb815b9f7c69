"""
The reference's own ``basic/bias.py`` (``BiasScorer``) and ``basic/popularity.py`` (``PopScorer``) on top of the
sandbox of ``ref_sandbox``; and the recording of both on ml-latest-small that
``tests/golden/reference_classes/basic_*.npz`` holds.
"""

from __future__ import annotations

import contextlib

import numpy as np
import pandas as pd

import ref_sandbox
from svd_ref_sandbox import SCORE_ITEMS, SCORE_USERS, UNKNOWN_ID, rated_query

#: the recorded BiasScorer configurations, by golden-file name
BIAS_CONFIGS = {
    "plain": {},
    "damped": {"damping": 5.0},
    "dict": {"damping": {"user": 2.0, "item": 7.5}},
    "items": {"entities": {"item"}, "damping": 3.0},
    "users": {"entities": {"user"}, "damping": 0.1},
}
POP_SCORES = ("quantile", "rank", "count")


class StatsDataset(ref_sandbox.FakeDataset):
    """``FakeDataset`` plus ``item_stats()``'s ``count`` column: int64 counts indexed by the item vocabulary's ids."""

    def item_stats(self) -> pd.DataFrame:
        counts = np.bincount(self._inter.items, minlength=self._inter.n_items).astype(np.int64)
        return pd.DataFrame({"count": counts}, index=pd.Index(self.items.ids(), name="item_id"))


@contextlib.contextmanager
def basic_modules():
    """``ref_sandbox.reference_modules()`` (which loads ``basic/bias.py``) plus ``basic/popularity.py``."""
    with ref_sandbox.reference_modules() as mods:
        mods["lenskit.basic.popularity"] = ref_sandbox._load("lenskit.basic.popularity", "basic/popularity.py")
        yield mods


def queries(ml_small):
    """``(user id, history ids or None, history ratings or None)`` of every scored query, in the golden files'
    order: the sampled users, an unknown user, a known and an unknown user with a rated history, and an unknown user
    whose history has no ratings."""
    u0 = int(SCORE_USERS[0])
    ids, ratings = rated_query(ml_small, u0)
    out = [(ml_small.user_ids[u], None, None) for u in SCORE_USERS]
    out.append((UNKNOWN_ID, None, None))
    out.append((ml_small.user_ids[u0], ids, ratings))
    out.append((UNKNOWN_ID, ids, ratings))
    out.append((UNKNOWN_ID, ids, None))
    return out


def score_item_ids(ml_small) -> np.ndarray:
    """The scored items: every 29th item, then an unknown one."""
    return np.append(ml_small.item_ids[SCORE_ITEMS], UNKNOWN_ID)


def record(ml_small) -> dict[str, dict]:
    """The reference classes trained on ml-latest-small, by golden-file name: each BiasScorer configuration's model
    and ``__call__`` scores, and each PopScorer mode's ``item_scores`` and ``__call__`` scores."""
    out = {}
    with basic_modules() as ref:
        bias, pop = ref["lenskit.basic.bias"], ref["lenskit.basic.popularity"]
        ItemList, RecQuery = ref["lenskit.data._items"].ItemList, ref["lenskit.data._query"].RecQuery
        data = StatsDataset(ml_small)
        items = ItemList(item_ids=score_item_ids(ml_small))
        for name, cfg in BIAS_CONFIGS.items():
            m = bias.BiasScorer(bias.BiasConfig(**cfg))
            m.train(data)
            scores = []
            for uid, hist, ratings in queries(ml_small):
                h = None if hist is None else ItemList(item_ids=hist, **({} if ratings is None else {"rating": ratings}))
                scores.append(np.asarray(m(RecQuery(user_id=uid, history_items=h), items).scores("numpy")))
            md = m.model
            out[f"basic_bias_{name}"] = {
                "global_bias": np.float64(md.global_bias),
                "item_biases": np.zeros(0, np.float32) if md.item_biases is None else md.item_biases,
                "user_biases": np.zeros(0, np.float32) if md.user_biases is None else md.user_biases,
                "has_items": np.bool_(md.item_biases is not None), "has_users": np.bool_(md.user_biases is not None),
                "scores": np.stack(scores),
            }  # fmt: skip
        for mode in POP_SCORES:
            m = pop.PopScorer(pop.PopConfig(score=mode))
            m.train(data)
            out[f"basic_pop_{mode}"] = {
                "item_scores": m.item_scores, "scores": np.asarray(m(items).scores("numpy")),
            }  # fmt: skip
    return out
