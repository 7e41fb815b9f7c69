"""
Stochastic top-n ranking on the H100 engine — the component surface of ``lenskit.stochastic.StochasticTopNRanker``
(``src/lenskit/stochastic/_ranker.py``): Plackett–Luce sampling of rankings by exponential keys, drawing NumPy's PCG64
stream exactly as the reference does.

Same config (:class:`StochasticTopNConfig`: ``n``, ``rng``, ``transform``, ``scale``) and the same ``__call__``;
plus ``rank_batch`` for many scored lists and ``rank_scores`` for a device score matrix, both on
``lk_stochastic_topn``.  For every list the valid items are those with a finite score; the k-th of them, in list
order, draws the k-th uniform of the query's generator, and its key is ``log(u) / max(w, smallest f32 normal)`` for
its weight ``w`` (softmax, linear or the scaled score).  The top ``n`` keys are selected by argtopn's heap, every key
sorted for ``n`` of None or negative.

The generators are the reference's ``derivable_rng`` (``src/lenskit/random.py:227-349``), restated here:

* a seed or None: one generator (``FixedRNG``) shared by every call, so consecutive calls continue one stream.  A
  batch draws for its lists in order from that stream on the device, and the host generator is then advanced by the
  batch's draws, which leaves it exactly where the sequence of calls would;
* ``"user"`` or ``(seed, "user")``: a generator per call (``DerivingRNG``), seeded from the base seed and the query's
  user id (``make_seed``, which hashes string ids with md5), or spawned from the base seed for a query without one.

This package has no global RNG, so ``rng=None`` is ``np.random.default_rng(None)``.
"""

from __future__ import annotations

from hashlib import md5
from typing import Literal

import numpy as np
import torch
from numpy.random import SeedSequence, default_rng
from pydantic import BaseModel

from . import _lib, engine
from .batch import check_exclude, history_csr, take
from .components import Component, ItemList, RecQuery

#: a configured seed: an int, a sequence of ints or None
ConfiguredSeed = int | list[int] | None
#: the ``rng`` of :class:`StochasticTopNConfig` (the reference's ``DerivableSeed``)
DerivableSeed = ConfiguredSeed | Literal["user"] | tuple[ConfiguredSeed, Literal["user"]]


class StochasticTopNConfig(BaseModel, extra="forbid"):
    n: int | None = None
    "The number of items to select; -1 or None for every valid item."
    rng: DerivableSeed = None
    transform: Literal["softmax", "linear"] | None = "softmax"
    scale: float = 1.0


# ---------------------------------------------------------------------------
# derivable RNGs (random.py:227-349)
# ---------------------------------------------------------------------------


def _bytes_seed(key: bytes) -> int:
    """The md5 digest as four int32 words, xor-ed together, absolute value."""
    words = np.frombuffer(md5(key).digest(), np.int32)
    return abs(int(np.bitwise_xor.reduce(words)))


def make_seed(*keys) -> SeedSequence:
    """A seed sequence whose entropy is the keys' material in order: a seed sequence's entropy, ints as they are,
    strings and bytes hashed by :func:`_bytes_seed`, sequences spliced in; None is skipped."""
    seed: list[int] = []
    for key in keys:
        if key is None:
            continue
        if isinstance(key, SeedSequence):
            if key.entropy is not None:
                seed += [key.entropy] if isinstance(key.entropy, int) else list(key.entropy)
        elif isinstance(key, (int, np.integer)):
            seed.append(int(key))
        elif isinstance(key, str):
            seed.append(_bytes_seed(key.encode("utf8")))
        elif isinstance(key, bytes):
            seed.append(_bytes_seed(key))
        elif hasattr(key, "bytes") and hasattr(key, "hex"):  # a UUID
            seed.append(_bytes_seed(key.bytes))
        else:
            seed += list(key)
    return SeedSequence(seed)


class FixedRNG:
    """Every query draws from the one generator ``rng``."""

    def __init__(self, rng: np.random.Generator):
        self.rng = rng

    def __call__(self, query: RecQuery | None = None) -> np.random.Generator:
        return self.rng


class DerivingRNG:
    """Each query gets a new generator: seeded from ``seed`` and its user id, or spawned from ``seed``."""

    def __init__(self, seed: SeedSequence):
        self.seed = seed

    def __call__(self, query: RecQuery | None = None) -> np.random.Generator:
        if query is None or query.user_id is None:
            return default_rng(self.seed.spawn(1)[0])
        return default_rng(make_seed(self.seed, query.user_id))


def derivable_rng(spec) -> FixedRNG | DerivingRNG:
    """``"user"``, ``(seed, "user")`` or a seed, as the reference reads them."""
    if isinstance(spec, str) and spec == "user":
        return DerivingRNG(SeedSequence())
    if isinstance(spec, tuple):
        seed, key = spec
        if key != "user":
            raise ValueError(f"unrecognized key {key}")
        return DerivingRNG(make_seed(seed))
    return FixedRNG(default_rng(spec))


def generator_words(gen: np.random.Generator) -> list[int]:
    """A PCG64 generator's ``(state, inc)`` as ``lk_stochastic_topn``'s four u64 words."""
    st = gen.bit_generator.state
    if st["bit_generator"] != "PCG64":
        raise TypeError(f"stochastic ranking draws NumPy's PCG64 stream, not {st['bit_generator']}")
    return engine.pcg64_words(st["state"]["state"], st["state"]["inc"])


def advance(gen: np.random.Generator, draws: int) -> None:
    """Leave ``gen`` where ``draws`` 64-bit draws (``uniform``) leave it: the LCG advanced, the buffered 32-bit half
    untouched."""
    bg = gen.bit_generator
    before = bg.state
    bg.advance(draws)
    after = bg.state
    after["has_uint32"], after["uinteger"] = before["has_uint32"], before["uinteger"]
    bg.state = after


# ---------------------------------------------------------------------------
# the ranker
# ---------------------------------------------------------------------------


class StochasticTopNRanker(Component):
    """
    ``StochasticTopNRanker``: ``__call__(items, query, n)`` samples a ranking of the list's valid items.
    :meth:`rank_batch` ranks many lists in one launch, :meth:`rank_scores` every item of a device score matrix.
    """

    CONFIG_CLASS = StochasticTopNConfig
    config: StochasticTopNConfig

    def __init__(self, config=None, **kwargs):
        super().__init__(config, **kwargs)
        self._rng_factory = derivable_rng(self.config.rng)

    def __call__(self, items: ItemList, query=None, n: int | None = None, *, include_weights: bool = False) -> ItemList:
        return self.rank_batch([items], [query], n, include_weights=include_weights)[0]

    def _n(self, n: int | None) -> int | None:
        """The call's ``n`` unless it is None or negative, else the config's (0 there means every item); None for
        every item."""
        if n is None or n < 0:
            n = self.config.n or -1
        return None if n < 0 else int(n)

    def _streams(self, queries: list[RecQuery]):
        """``(states [1 or B, 4] u64, shared, the shared generator or None)``; the factory is asked once per query
        in order, as the calls would."""
        f = self._rng_factory
        if isinstance(f, FixedRNG):
            return np.array([generator_words(f.rng)], dtype=np.uint64), True, f.rng
        return np.array([generator_words(f(q)) for q in queries], dtype=np.uint64).reshape(-1, 4), False, None

    def _run(self, scores: torch.Tensor, queries: list[RecQuery], n: int | None, include_weights: bool, excl=(None, None)):
        states, shared, gen = self._streams(queries)
        # n = 0 still draws for every list with valid items (the reference computes the keys, then takes none)
        idx, val, key, cnt, drawn = engine.stochastic_topn(
            scores, 1 if n == 0 else n, transform=self.config.transform, scale=self.config.scale, states=states,
            shared=shared, excl_indptr=excl[0], excl_items=excl[1], with_keys=include_weights,
        )  # fmt: skip
        if gen is not None:
            advance(gen, int(drawn.item()))
        if n == 0:
            cnt = torch.zeros_like(cnt)
        host = lambda t: None if t is None else t.cpu().numpy()  # noqa: E731
        return host(idx), host(val), host(key), host(cnt)

    def rank_batch(self, lists: list[ItemList], queries=None, n: int | None = None, *,
                   include_weights: bool = False) -> list[ItemList]:  # fmt: skip
        """
        ``[self(items, query, n) for items, query in zip(lists, queries)]`` in one launch: the lists' scores are
        packed into a NaN-padded device matrix.  Under a fixed generator the lists draw from its stream in order, and
        the generator ends where those calls would leave it.  Each result keeps its list's fields, with ``weight``
        (the keys) when ``include_weights``.
        """
        queries = [RecQuery.create(q) for q in (queries if queries is not None else [None] * len(lists))]
        if len(queries) != len(lists):
            raise ValueError(f"{len(lists)} lists and {len(queries)} queries")
        host = []
        for items in lists:
            s = items.scores()
            if s is None:
                raise ValueError("item list must have scores")
            host.append(np.asarray(s, dtype=np.float32))
        L = max((len(s) for s in host), default=0)
        packed = np.full((len(host), L), np.nan, dtype=np.float32)
        for b, s in enumerate(host):
            packed[b, : len(s)] = s
        dev = _lib.require_device()
        idx, _val, key, cnt = self._run(torch.from_numpy(packed).to(dev), queries, self._n(n), include_weights)
        out = []
        for b, items in enumerate(lists):
            c = int(cnt[b])
            extra = {"weight": key[b, :c].copy()} if include_weights else {}
            out.append(take(items, idx[b, :c].astype(np.int64), **extra))
        return out

    def rank_scores(self, scores: torch.Tensor, queries, vocabulary, n: int | None = None, *,
                    exclude: Literal["query"] | None = "query", include_weights: bool = False) -> list[ItemList]:  # fmt: skip
        """
        Rank every item of ``vocabulary`` for each query from the device matrix ``scores`` [B, n_items] (f32, any
        strides, such as ``scorer.score_matrix(queries).T``), without copying it to the host.  Query b's list is
        every item in vocabulary order with the scores of row b, minus its ``query_items`` when ``exclude="query"``
        (what ``TrainingItemsCandidateSelector`` gives); items with a non-finite score, such as the whole row of an
        unscorable query, are left out.  Returns ``ItemList``s with ``score`` (and ``weight``).
        """
        check_exclude(exclude)
        queries = [RecQuery.create(q) for q in queries]
        if scores.dim() != 2 or scores.shape[0] != len(queries) or scores.shape[1] != len(vocabulary):
            raise ValueError(f"scores must be [{len(queries)}, {len(vocabulary)}], not {list(scores.shape)}")
        excl = history_csr(queries, vocabulary, scores.device)[1:] if exclude == "query" else (None, None)
        idx, val, key, cnt = self._run(scores, queries, self._n(n), include_weights, excl)
        out = []
        for b in range(len(queries)):
            c = int(cnt[b])
            nums = idx[b, :c].copy()
            extra = {"weight": key[b, :c].copy()} if include_weights else {}
            out.append(ItemList(item_ids=vocabulary.ids(nums), item_nums=nums, vocabulary=vocabulary,
                                scores=val[b, :c].copy(), **extra))  # fmt: skip
        return out
