"""
Minimal stand-ins for the reference types the two scorers touch.

The real ``lenskit`` package is not importable in this image (its Rust extension
is not built), so the scorers in ``lkpy_b200.als`` / ``lkpy_b200.knn`` are written
against these small classes, which keep the names and call shapes of

* ``Vocabulary``        (``src/lenskit/data/_vocab.py``)
* ``ItemList``          (``src/lenskit/data/_items.py``) — ids / numbers / fields / scores
* ``RecQuery``          (``src/lenskit/data/_query.py``)
* ``TrainingOptions``   (``src/lenskit/training.py:42-149``)
* ``Component`` / ``Trainable`` / ``UsesTrainer`` / ``ModelTrainer``
                        (``src/lenskit/pipeline/components.py:65-199``, ``training.py:231-378``)

INTEGRATION.md shows how the same engines bind under the real classes.
"""

from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Literal

import numpy as np

from .data import Interactions


class Vocabulary:
    """Sorted id <-> number map."""

    def __init__(self, ids, name: str | None = None):
        self._ids = np.asarray(ids)
        self.name = name
        self._sorted = bool(np.all(self._ids[:-1] < self._ids[1:])) if len(self._ids) > 1 else True
        self._index = None if self._sorted else {v: i for i, v in enumerate(self._ids.tolist())}

    @property
    def size(self) -> int:
        return len(self._ids)

    def __len__(self) -> int:
        return len(self._ids)

    def ids(self, numbers=None) -> np.ndarray:
        return self._ids if numbers is None else self._ids[np.asarray(numbers)]

    def id(self, number: int):
        return self._ids[number]

    def numbers(self, ids, missing: Literal["error", "negative"] = "error") -> np.ndarray:
        ids = np.asarray(ids)
        if self._sorted:
            pos = np.searchsorted(self._ids, ids)
            pos = np.minimum(pos, max(len(self._ids) - 1, 0))
            ok = (self._ids[pos] == ids) if len(self._ids) else np.zeros(len(ids), bool)
            out = np.where(ok, pos, -1).astype(np.int32)
        else:
            out = np.array([self._index.get(v, -1) for v in ids.tolist()], dtype=np.int32)
        if missing == "error" and np.any(out < 0):
            raise KeyError("unknown ids")
        return out

    def number(self, id_, missing: Literal["error", "none"] | None = "error"):
        n = int(self.numbers([id_], missing="negative")[0])
        if n < 0:
            if missing == "error":
                raise KeyError(id_)
            return None
        return n

    def __eq__(self, other) -> bool:
        return isinstance(other, Vocabulary) and np.array_equal(self._ids, other._ids)


class ItemList:
    """Items identified by id and/or number, with named fields (``rating``, ``score`` …).  ``ordered`` marks a
    ranked list; a copy keeps its source's flag unless given one."""

    def __init__(self, items=None, *, item_ids=None, item_nums=None, vocabulary: Vocabulary | None = None,
                 scores=None, ordered: bool | None = None, **fields):
        self.ordered = bool(ordered)
        if isinstance(items, ItemList):
            if ordered is None:
                self.ordered = items.ordered
            item_ids, item_nums = items._ids, items._nums
            vocabulary = vocabulary or items._vocab
            base = dict(items._fields)
            base.pop("score", None)
            base.update(fields)
            fields = base
        elif items is not None:
            item_ids = np.asarray(items)
        self._ids = None if item_ids is None else np.asarray(item_ids)
        self._nums = None if item_nums is None else np.asarray(item_nums, dtype=np.int32)
        self._vocab = vocabulary
        n = len(self)
        self._fields: dict[str, np.ndarray] = {}
        for k, v in fields.items():
            self._fields[k] = self._col(v, n)
        if scores is not None:
            self._fields["score"] = self._col(scores, n, np.float32)

    @staticmethod
    def _col(v, n, dtype=None):
        a = np.asarray(v, dtype=dtype)
        if a.ndim == 0:
            a = np.full(n, a, dtype=a.dtype)
        if len(a) != n:
            raise ValueError("field length mismatch")
        return a

    def __len__(self) -> int:
        if self._ids is not None:
            return len(self._ids)
        return 0 if self._nums is None else len(self._nums)

    def ids(self) -> np.ndarray:
        if self._ids is None:
            assert self._vocab is not None and self._nums is not None
            self._ids = self._vocab.ids(self._nums)
        return self._ids

    def numbers(self, format: str = "numpy", *, vocabulary: Vocabulary | None = None,
                missing: Literal["error", "negative"] = "error") -> np.ndarray:
        if vocabulary is None or vocabulary is self._vocab or (self._vocab is not None and vocabulary == self._vocab):
            if self._nums is not None:
                return self._nums
            vocabulary = vocabulary or self._vocab
        if vocabulary is None:
            raise RuntimeError("item numbers need a vocabulary")
        return vocabulary.numbers(self.ids(), missing=missing)

    def field(self, name: str, format: str = "numpy"):
        return self._fields.get(name)

    def scores(self):
        return self._fields.get("score")

    def to_df(self):
        import pandas as pd

        d = {"item_id": self.ids()}
        d.update(self._fields)
        return pd.DataFrame(d)


@dataclass
class RecQuery:
    user_id: Any = None
    query_items: ItemList | None = None

    @classmethod
    def create(cls, q) -> "RecQuery":
        if isinstance(q, RecQuery):
            return q
        if isinstance(q, ItemList):
            return cls(None, q)
        return cls(q, None)


@dataclass
class TrainingOptions:
    """``lenskit.training.TrainingOptions`` (training.py:42-149): retrain / device / rng."""

    retrain: bool = True
    device: str | None = None
    rng: Any = None

    def random_generator(self) -> np.random.Generator:
        if isinstance(self.rng, np.random.Generator):
            return self.rng
        return np.random.default_rng(self.rng)


class Component:
    """``lenskit.pipeline.Component``: config object + ``__call__``."""

    config: Any
    CONFIG_CLASS: type | None = None

    def __init__(self, config=None, **kwargs):
        cls = self.CONFIG_CLASS
        if config is None and cls is not None:
            config = cls(**kwargs)
        elif isinstance(config, dict) and cls is not None:
            config = cls(**config)
        elif kwargs:
            raise TypeError("pass either a config object or keyword options")
        self.config = config

    def dump_config(self) -> dict:
        return self.config.model_dump()


class Trainable:
    def train(self, data, options: TrainingOptions = TrainingOptions()) -> None:  # pragma: no cover
        raise NotImplementedError

    def is_trained(self) -> bool:  # pragma: no cover
        raise NotImplementedError


class ModelTrainer:
    """``lenskit.training.ModelTrainer`` (training.py:337-378)."""

    def train_epoch(self) -> dict[str, float] | None:  # pragma: no cover
        raise NotImplementedError

    def finalize(self) -> None:  # pragma: no cover
        raise NotImplementedError


class UsesTrainer(Trainable):
    """``lenskit.training.UsesTrainer.train`` (training.py:301-334): epoch loop over a trainer."""

    def create_trainer(self, data, options: TrainingOptions) -> ModelTrainer:  # pragma: no cover
        raise NotImplementedError

    def train(self, data, options: TrainingOptions = TrainingOptions()) -> None:
        if self.is_trained() and not options.retrain:
            return
        trainer = self.create_trainer(data, options)
        self.training_log: list[dict] = []
        for _i in range(1, self.config.epochs + 1):
            metrics = trainer.train_epoch()
            self.training_log.append(metrics or {})
        trainer.finalize()


@dataclass
class Dataset:
    """The slice of ``lenskit.data.Dataset`` the two scorers use, plus optional per-item attributes (name -> one
    value per item of ``items``, in vocabulary order), which ``FAIRReranker`` reads its protected flags from."""

    interactions: Any  # lkpy_b200.data.Interactions
    users: Vocabulary = field(default=None)  # type: ignore[assignment]
    items: Vocabulary = field(default=None)  # type: ignore[assignment]
    item_attributes: dict[str, Any] = field(default_factory=dict)

    def __post_init__(self):
        it = self.interactions
        if self.users is None:
            self.users = Vocabulary(it.user_ids if it.user_ids is not None else np.arange(it.n_users), "user")
        if self.items is None:
            self.items = Vocabulary(it.item_ids if it.item_ids is not None else np.arange(it.n_items), "item")

    @property
    def user_count(self) -> int:
        return self.interactions.n_users

    @property
    def item_count(self) -> int:
        return self.interactions.n_items

    def user_history(self, user_num: int) -> ItemList:
        """What ``UserTrainingHistoryLookup`` returns (``basic/history.py``)."""
        it = self.interactions
        lo, hi = np.searchsorted(it.users, [user_num, user_num + 1])
        return ItemList(item_nums=it.items[lo:hi], vocabulary=self.items, rating=it.ratings[lo:hi])


def _as_dataset(data) -> Dataset:
    if isinstance(data, Dataset):
        return data
    if isinstance(data, Interactions):
        return Dataset(data)
    raise TypeError("expected a Dataset or Interactions")
