"""
NMF scorer on the H100 engine — the component surface of ``lenskit.sklearn.nmf.NMFScorer``
(``src/lenskit/sklearn/nmf.py``): scikit-learn's ``non_negative_factorization`` of the user x item indicator matrix.

Same config (``max_iter`` / ``epochs``, ``embedding_size`` / ``n_components`` / ``embedding_size_exp``,
``beta_loss``, ``alpha_W``, ``alpha_H``, ``l1_ratio``, ``method``), the same trained attributes (``users``,
``items``, ``user_components`` [n_users, k] and ``item_components`` [n_items, k], host f32) and the same
``__call__``; plus ``n_iter_``, ``score_matrix``, ``score_batch`` and ``recommend_batch``.

Training follows scikit-learn (``solver="cd"``, ``init=None``, ``tol=1e-4``, no shuffling) on the device:

* the initialisation: ``nndsvda`` when k <= min(n_users, n_items), on :func:`engine.randomized_svd_usv` (the start
  matrix drawn from NumPy's global ``RandomState``) and :func:`engine.nndsvd`; else ``"random"``, drawn on the host
  from the global ``RandomState`` in scikit-learn's order.  Under ``np.random.seed`` the draws are the reference's and
  the global state is left where the reference leaves it.  ``X.mean()`` is SciPy's;
* each iteration: ``X @ Ht`` and ``Xᵀ @ W`` on ``lk_spmm`` (exact: X holds ones), the Grams in f64 rounded once to
  f32 (scikit-learn's are f32 sgemms), the sweeps on ``lk_nmf_cd_sweep`` (``_update_cdnmf_fast`` bit for bit) and
  the two violations on ``lk_f32_seq_sum`` (its f32 sum bit for bit), then scikit-learn's stopping test on the host;
* ``ConvergenceWarning`` when ``max_iter`` is reached.

The SVD of the initialisation is cuSOLVER's instead of LAPACK's and the Grams are rounded once, so the factors agree
with the reference's to rounding, not bit for bit (DESIGN.md §4.17).

Scoring is the known-user path of :class:`factors.KnownUserScorer` (``lk_als_recommend_batch``) over
``user_components`` and ``item_components`` with no offsets: one f32 FMA chain per score, where the reference takes an
f32 product and returns it as f64.
"""

from __future__ import annotations

import warnings
from typing import Literal

import numpy as np
import scipy.sparse as sps
import torch
from pydantic import AliasChoices, Field, PositiveInt, field_validator

from . import _lib, engine
from .components import Trainable, TrainingOptions, _as_dataset
from .factors import EmbeddingSizeExp, KnownUserScorer, within_engine_limit
from .prep import coo_to_csr_pair

try:
    from sklearn.exceptions import ConvergenceWarning
except ImportError:  # scikit-learn is the reference's dependency, not this package's

    class ConvergenceWarning(UserWarning):
        """scikit-learn's warning that an iterative solver stopped at its iteration limit."""


#: scikit-learn's ``_randomized_svd`` default ``n_oversamples`` and NMF's ``tol``
N_OVERSAMPLES = 10
TOL = 1e-4


class NMFConfig(EmbeddingSizeExp, extra="forbid"):
    beta_loss: Literal["frobenius", "kullback-leibler", "itakura-saito"] = "frobenius"
    max_iter: PositiveInt = Field(default=200, validation_alias=AliasChoices("max_iter", "epochs"))
    embedding_size: PositiveInt | None = Field(
        default=64, validation_alias=AliasChoices("embedding_size", "n_components")
    )
    alpha_W: float = 0.0
    alpha_H: float | Literal["same"] = "same"
    l1_ratio: float = 0.0
    method: Literal["full", "minibatch"] = "full"

    @field_validator("embedding_size", mode="after")
    @staticmethod
    def check_embedding_size(k) -> int:
        if k is None:
            raise ValueError("embedding_size=None (scikit-learn's n_features) is not covered by the engine")
        return within_engine_limit(k)

    @field_validator("beta_loss", mode="after")
    @staticmethod
    def check_beta_loss(beta_loss) -> str:
        if beta_loss != "frobenius":
            raise ValueError(f"beta_loss={beta_loss!r}: the coordinate-descent solver supports only 'frobenius'")
        return beta_loss

    @field_validator("method", mode="after")
    @staticmethod
    def check_method(method) -> str:
        if method == "minibatch":
            raise ValueError("method='minibatch' (scikit-learn's MiniBatchNMF) is not covered by the engine")
        return method

    def regularization(self, n_rows: int, n_cols: int) -> tuple[float, float, float, float]:
        """scikit-learn's ``_compute_regularization``: ``(l1_reg_W, l1_reg_H, l2_reg_W, l2_reg_H)``."""
        alpha_W = self.alpha_W
        alpha_H = self.alpha_W if self.alpha_H == "same" else self.alpha_H
        return (n_cols * alpha_W * self.l1_ratio, n_rows * alpha_H * self.l1_ratio,
                n_cols * alpha_W * (1.0 - self.l1_ratio), n_rows * alpha_H * (1.0 - self.l1_ratio))  # fmt: skip


def indicator_operand(users: np.ndarray, items: np.ndarray, n_users: int, n_items: int, dev) -> engine.SvdOperand:
    """The indicator matrix X [n_users, n_items] (f32 ones) in HBM, both orientations; COO sorted by (user, item)."""
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    ones = torch.ones(len(users), dtype=torch.float32, device=dev)
    ui, iu, _perm = coo_to_csr_pair(up(users), up(items), ones, n_users, n_items)
    return engine.SvdOperand.create(ui, iu)


def indicator_mean(x: engine.SvdOperand) -> np.float32:
    """SciPy's ``X.mean()`` of the f32 indicator matrix."""
    m = x.rows
    ones = np.ones(m.nnz, dtype=np.float32)
    return sps.csr_matrix((ones, m.indices.cpu().numpy(), m.h_indptr), shape=m.shape).mean()


def initialize(x: engine.SvdOperand, k: int, stage=None) -> tuple[torch.Tensor, torch.Tensor]:
    """scikit-learn's ``_initialize_nmf(X, k, init=None)``: W [n_rows, k] and H [k, n_cols] on the device."""
    n_rows, n_cols = x.shape
    dev = x.rows.indptr.device
    mean = indicator_mean(x)
    if k > min(n_rows, n_cols):  # init="random": H drawn before W
        avg = np.sqrt(mean / k)
        H = np.abs(avg * np.random.standard_normal(size=(k, n_cols)).astype(np.float32))
        W = np.abs(avg * np.random.standard_normal(size=(n_rows, k)).astype(np.float32))
        return torch.from_numpy(W).to(dev), torch.from_numpy(H).to(dev)
    n_iter = 7 if k < 0.1 * min(n_rows, n_cols) else 4  # n_iter="auto"
    q0 = np.random.normal(size=(min(n_rows, n_cols), k + N_OVERSAMPLES)).astype(np.float32)
    u, s, vt = engine.randomized_svd_usv(x, torch.from_numpy(q0).to(dev), k, n_iter, stage)
    return engine.nndsvd(u, s, vt, float(mean))


def factorize(x: engine.SvdOperand, config: NMFConfig, stage=None) -> tuple[torch.Tensor, torch.Tensor, int]:
    """``non_negative_factorization(X, ...)`` with the configuration's options on the device: ``(W, H, n_iter)``,
    W [n_rows, k] and H [k, n_cols] in HBM."""
    k = config.embedding_size
    W, H = initialize(x, k, stage)
    l1_W, l1_H, l2_W, l2_H = config.regularization(*x.shape)
    d = engine.NmfDescent(x, W, H.T.contiguous(), l1_W, l1_H, l2_W, l2_H)
    violation_init = None
    n_iter = 0
    for n_iter in range(1, config.max_iter + 1):
        v_W, v_H = d.iteration(stage)
        violation = 0.0
        violation += v_W
        violation += v_H
        if n_iter == 1:
            violation_init = violation
        if violation_init == 0:
            break
        if violation / violation_init <= TOL:
            break
    if n_iter == config.max_iter:
        warnings.warn(f"Maximum number of iterations {config.max_iter} reached. Increase it to improve convergence.",
                      ConvergenceWarning, stacklevel=2)  # fmt: skip
    return d.W, d.Ht.T, n_iter


class NMFScorer(KnownUserScorer, Trainable):
    """
    ``NMFScorer``: ``train`` on the device, and the known-user scoring of :class:`KnownUserScorer`
    (``score_matrix`` / ``score_batch`` / ``__call__`` / ``recommend_batch``) with no offsets.  A query whose user
    is unknown scores NaN and gets an empty list.
    """

    CONFIG_CLASS = NMFConfig
    config: NMFConfig

    user_components: np.ndarray | None = None
    item_components: np.ndarray | None = None
    n_iter_: int | None = None

    def is_trained(self) -> bool:
        return self.item_components is not None

    def train(self, data, options: TrainingOptions = TrainingOptions()) -> None:
        if self.is_trained() and not options.retrain:
            return
        ds = _as_dataset(data)
        dev = _lib.require_device()
        it = ds.interactions
        x = indicator_operand(it.users, it.items, it.n_users, it.n_items, dev)
        W, H, self.n_iter_ = factorize(x, self.config)
        self.user_components = W.cpu().numpy()
        self.item_components = np.ascontiguousarray(H.T.cpu().numpy())
        self.users, self.items = ds.users, ds.items
        self.user_embeddings = self.user_components
        self.item_embeddings = self.item_components
