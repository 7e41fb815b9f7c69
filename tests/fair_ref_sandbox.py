"""
The reference's own ``reranking/fair.py`` (``FAIRReranker``) on top of the sandbox of ``ref_sandbox``; and the
recording of its thresholds and calls that ``tests/golden/reference_classes/fair_*.npz`` holds.

The reference trains from ``Dataset.entities("item")``; ``_Entities`` below is that slice (``attributes``,
``attribute(name).numpy()``, ``vocabulary``) over the reference's own ``Vocabulary``.  Everything else, from the
configuration to the re-ranked ``ItemList``, is the reference's code.
"""

from __future__ import annotations

import contextlib

import numpy as np

import ref_sandbox

#: ``(n, p, alpha)`` of the recorded thresholds: the reference tests' cases, n = 1 and 1000, p of 0.1 and 0.9, and
#: (4, 0.1, 0.05) and (3, 0.05, 0.1), whose m_list is all zero
THRESHOLDS = [
    (9, 0.5, 0.1), (10, 0.5, 0.1), (4, 0.9, 1e-10), (1, 0.5, 0.1), (1000, 0.5, 0.1), (20, 0.5, 0.2), (50, 0.5, 0.1),
    (100, 0.1, 0.3), (150, 0.9, 0.1), (20, 0.1, 0.1), (20, 0.9, 0.1), (64, 0.7, 0.05), (5, 0.1, 0.05),
    (4, 0.1, 0.05), (3, 0.05, 0.1),
]  # fmt: skip

#: the recorded re-rankers, by golden-file name: their config and the item vocabulary's size
CASES = {
    "fair_calls_n10": {"n": 10, "p": 0.5, "alpha": 0.1},
    "fair_calls_n40": {"n": 40, "p": 0.7, "alpha": 0.1, "protected_attribute": "flag"},
    "fair_calls_extreme": {"n": 4, "p": 0.9, "alpha": 1e-10},
    "fair_calls_zero": {"n": 4, "p": 0.1, "alpha": 0.05},
}
N_ITEMS = 120
#: the ``n`` of a call that passes none
NONE_N = -999


def vocabulary(name: str):
    """``(item ids, protected flags)`` of case ``name``'s training data: ids 100, 103, ... and about a third of them
    protected."""
    rng = np.random.default_rng(sum(map(ord, name)))
    return np.arange(N_ITEMS, dtype=np.int64) * 3 + 100, rng.random(N_ITEMS) < 0.35


def calls(name: str) -> list[tuple[np.ndarray, int | None]]:
    """``(list ids, n)`` of every recorded call of case ``name``: lists with unknown items, none and only protected
    items, lists shorter than the config's n, a runtime n below, equal to and 0 against it, and protected items
    deep in a list that the constraint pulls forward.  No empty list: the reference raises ``TypeError`` on one (an
    empty index list has no Arrow type), where this package returns an empty list."""
    ids, prot = vocabulary(name)
    nc = CASES[name]["n"]
    rng = np.random.default_rng(7 + sum(map(ord, name)))
    out: list[tuple[np.ndarray, int | None]] = []
    for n in (None, nc, nc // 2, 0, 1):
        out.append((rng.permutation(ids)[: 2 * nc + 5], n))
    mixed = rng.permutation(ids)[: nc + 8].copy()
    mixed[::3] = 10_000 + np.arange(len(mixed[::3]))  # ids outside the vocabulary: unprotected
    out.append((mixed, None))
    out.append((rng.permutation(ids[~prot])[: nc + 3], None))  # no protected item
    out.append((rng.permutation(ids[prot])[: nc + 3], None))  # only protected items
    out.append((rng.permutation(ids)[: max(nc // 2, 1)], None))  # shorter than n
    out.append((rng.permutation(ids)[:1], None))
    # every unprotected item first, the protected ones deep in the list
    out.append((np.concatenate([rng.permutation(ids[~prot]), rng.permutation(ids[prot])]), None))
    out.append((np.concatenate([rng.permutation(ids[~prot])[: 3 * nc], rng.permutation(ids[prot])[:nc]]), nc - 1))
    return out


class _Attribute:
    def __init__(self, values):
        self._values = values

    def numpy(self):
        return self._values


class _Entities:
    """``Dataset.entities("item")`` as fair.py reads it."""

    def __init__(self, vocab, attrs: dict):
        self.vocabulary, self._attrs = vocab, attrs

    @property
    def attributes(self):
        return list(self._attrs)

    def attribute(self, name: str):
        return _Attribute(self._attrs[name])


class _Dataset:
    def __init__(self, vocab, attrs: dict):
        self._items = _Entities(vocab, attrs)

    def entities(self, kind: str):
        assert kind == "item"
        return self._items


@contextlib.contextmanager
def fair_modules():
    """``ref_sandbox.reference_modules()`` plus ``reranking/fair.py``."""
    with ref_sandbox.reference_modules() as mods:
        ref_sandbox._module("lenskit.reranking", package=True)
        mods["lenskit.reranking.fair"] = ref_sandbox._load("lenskit.reranking.fair", "reranking/fair.py")
        yield mods


def record() -> dict[str, dict]:
    """``fair_thresholds``: ``alpha_c`` and ``m_list`` of every ``THRESHOLDS`` entry.  Each ``CASES`` entry: its
    training data, ``alpha_c``, ``m_list`` and every call's list and chosen ids."""
    out = {}
    with fair_modules() as ref:
        fair, Vocabulary = ref["lenskit.reranking.fair"], ref["lenskit.data._vocab"].Vocabulary
        ItemList = ref["lenskit.data._items"].ItemList
        empty = _Dataset(Vocabulary(np.arange(1), "item"), {"protected": np.zeros(1, bool)})
        ac, mptr, ms = [], [0], []
        for n, p, alpha in THRESHOLDS:
            r = fair.FAIRReranker(fair.FAIRRerankerConfig(n=n, p=p, alpha=alpha))
            r.train(empty)
            ac.append(r.alpha_c)
            ms.append(np.asarray(r.m_list, np.int64))
            mptr.append(mptr[-1] + n)
        th = np.array(THRESHOLDS, dtype=np.float64)
        out["fair_thresholds"] = {"n": th[:, 0].astype(np.int64), "p": th[:, 1], "alpha": th[:, 2],
                                  "alpha_c": np.array(ac), "m_ptr": np.array(mptr), "m_list": np.concatenate(ms)}  # fmt: skip
        for name, cfg in CASES.items():
            ids, prot = vocabulary(name)
            attr = cfg.get("protected_attribute", "protected")
            r = fair.FAIRReranker(fair.FAIRRerankerConfig(**cfg))
            r.train(_Dataset(Vocabulary(ids, "item"), {attr: prot}))
            cs = calls(name)
            lptr, lists, optr, outs = [0], [], [0], []
            for items, n in cs:
                res = r(ItemList(item_ids=items, ordered=True), n)
                assert res.ordered
                got = np.asarray(res.ids(), np.int64)
                lists.append(items)
                lptr.append(lptr[-1] + len(items))
                outs.append(got)
                optr.append(optr[-1] + len(got))
            out[name] = {
                "vocab": ids, "protected": prot, "alpha_c": np.array(r.alpha_c), "m_list": np.asarray(r.m_list, np.int64),
                "list_ptr": np.array(lptr), "lists": np.concatenate(lists).astype(np.int64),
                "n": np.array([NONE_N if n is None else n for _i, n in cs]),
                "out_ptr": np.array(optr), "out": np.concatenate(outs),
            }  # fmt: skip
    return out

