"""
BiasedSVD scorer on the H100 engine — the component surface of ``lenskit.sklearn.svd.BiasedSVDScorer``
(``src/lenskit/sklearn/svd.py``): a bias model, then a truncated SVD of the bias residuals.

Same config (``embedding_size`` with the aliases ``features`` and ``embedding_size_exp``, ``damping``,
``algorithm``, ``n_iter``), the same trained attributes (``bias``, ``users``, ``items``, ``user_components``,
``components_``, ``singular_values_``, host f32 arrays) and the same ``__call__``; plus ``score_matrix``,
``score_batch`` and ``recommend_batch``.

Training follows the reference on the device:

* the bias model (``BiasModel.learn`` on the f32 ratings, on the host) and the residuals ``((r - g) - ib[item]) - ub[user]``, one f32
  rounding per step, computed on the device for the two CSR orientations;
* ``TruncatedSVD(algorithm="randomized", n_iter=n_iter).fit_transform``: the start matrix is drawn from NumPy's
  global ``RandomState``, as scikit-learn draws it with ``random_state=None`` (``TrainingOptions.rng`` is not used,
  as in the reference), so under ``np.random.seed`` the draws are the reference's and the global state is left
  where the reference leaves it.  The sparse products are ``lk_spmm`` (SciPy's products bit for bit) and the LU, QR
  and SVD are torch's on the device (cuSOLVER, f32) in place of SciPy's LAPACK on the host, so the factors agree to
  rounding, not bit for bit (DESIGN.md §4.16);
* ``user_components = X @ components_.T``, one more ``lk_spmm``.

``algorithm="arpack"`` (SciPy's ``svds``) is rejected when the configuration is made.

Scoring is the known-user path of :class:`factors.KnownUserScorer` (``lk_als_recommend_batch``): the user's component
row against ``components_.T``, with ``f32(g) + ib`` as the item offset and the user bias as the query offset, or the
bias of the query's ratings when the query carries rated items (:meth:`basic.BiasModel.user_bias_for_items`). Each
score is one f32 FMA chain over the components followed by two f32 adds; the reference computes ``user_components[u] @
components_`` as an f32 product and adds the biases in f64, returning f64 scores, so the two agree to f32 rounding.
"""

from __future__ import annotations

from typing import Literal

import numpy as np
import torch
from pydantic import AliasChoices, Field, NonNegativeFloat, NonNegativeInt, field_validator

from . import _lib, engine
from .basic import BiasModel
from .components import RecQuery, Trainable, TrainingOptions, _as_dataset
from .factors import EmbeddingSize, EmbeddingSizeExp, KnownUserScorer
from .prep import coo_to_csr_pair

#: scikit-learn's ``TruncatedSVD`` default ``n_oversamples``
N_OVERSAMPLES = 10


class BiasedSVDConfig(EmbeddingSizeExp, extra="forbid"):
    embedding_size: EmbeddingSize = Field(default=64, validation_alias=AliasChoices("embedding_size", "features"))
    damping: NonNegativeFloat | dict[Literal["user", "item"], NonNegativeFloat] = 5
    algorithm: Literal["arpack", "randomized"] = "randomized"
    n_iter: NonNegativeInt = 5

    @field_validator("algorithm", mode="after")
    @staticmethod
    def check_algorithm(algorithm) -> str:
        if algorithm == "arpack":
            raise ValueError("algorithm='arpack' (SciPy svds) is not covered by the engine (DESIGN.md §6)")
        return algorithm


class BiasedSVDScorer(KnownUserScorer, Trainable):
    """
    ``BiasedSVDScorer``: ``train`` on the device, and the known-user scoring of :class:`KnownUserScorer`
    (``score_matrix`` / ``score_batch`` / ``__call__`` / ``recommend_batch``) with the biases as the kernel's offsets.
    A query whose user is unknown scores NaN and gets an empty list.
    """

    CONFIG_CLASS = BiasedSVDConfig
    config: BiasedSVDConfig

    bias: BiasModel
    user_components: np.ndarray | None = None
    components_: np.ndarray | None = None
    singular_values_: np.ndarray | None = None

    def is_trained(self) -> bool:
        return self.components_ is not None

    def train(self, data, options: TrainingOptions = TrainingOptions()) -> None:
        if self.is_trained() and not options.retrain:
            return
        ds = _as_dataset(data)
        dev = _lib.require_device()
        it = ds.interactions
        k = self.config.embedding_size
        if it.n_items < 2:
            raise ValueError(f"Found array with {it.n_items} feature(s) while a minimum of 2 is required.")
        if k > it.n_items:
            raise ValueError(f"n_components({k}) must be <= n_features({it.n_items}).")
        self.bias = BiasModel.learn(it, self.config.damping, np.float32)  # the reference's f32 rating matrix
        x = residual_operand(self.bias, it, dev)
        # scikit-learn's draw: RandomState.normal from the global state, shape [M.shape[1], k + oversamples]
        q0 = np.random.normal(size=(min(it.n_users, it.n_items), k + N_OVERSAMPLES)).astype(np.float32)
        vt, s = engine.randomized_svd(x, torch.from_numpy(q0).to(dev), k, self.config.n_iter)
        self.components_ = vt.cpu().numpy()
        self.singular_values_ = s.cpu().numpy()
        self.user_components = x.mul(vt.T.contiguous()).cpu().numpy()
        self.users, self.items = ds.users, ds.items
        # the scoring path's tables: user rows, and item rows [n_items, k]
        self.user_embeddings = self.user_components
        self.item_embeddings = np.ascontiguousarray(self.components_.T)

    def embed_batch(self, queries):
        """Known users' embeddings, and as the user offset the bias of the query's ratings where it has them."""
        queries = [RecQuery.create(q) for q in queries]
        X, scorable, user_nums, _ = super().embed_batch(queries)
        fold_bias = np.full(len(queries), np.nan, dtype=np.float32)
        for b, q in enumerate(queries):
            ratings = None if q.query_items is None else q.query_items.field("rating")
            if ratings is not None:
                nums = q.query_items.numbers(vocabulary=self.items, missing="negative")
                fold_bias[b] = self.bias.user_bias_for_items(nums, ratings)
        return X, scorable, user_nums, fold_bias

    def batch_offsets(self, user_nums: np.ndarray, fold_bias):
        return self.bias.batch_offsets(user_nums, fold_bias)


def residual_operand(bias: BiasModel, it, dev) -> engine.SvdOperand:
    """The residual matrix X [n_users, n_items] in HBM, both orientations: ``((r - f32(g)) - ib[i]) - ub[u]``, each
    step an f32 subtraction as the reference's NumPy statements on the f32 rating array."""
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    users, items = up(it.users), up(it.items)
    vals = up(np.asarray(it.ratings, dtype=np.float32))
    vals = vals - float(np.float32(bias.global_bias))
    vals = vals - up(bias.item_biases)[items.long()]
    vals = vals - up(bias.user_biases)[users.long()]
    ui, iu, _perm = coo_to_csr_pair(users, items, vals, it.n_users, it.n_items)
    return engine.SvdOperand.create(ui, iu)
