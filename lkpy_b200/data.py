"""
Interaction-matrix inputs for the ALS / item-kNN hot paths.

Two sources, both host-side (NumPy) and both setup rather than hot path:

* ``load_ml_small()`` — the reference's vendored ``ml-latest-small`` ratings
  (LensKit's ``data/ml-latest-small/ratings.csv``, stored as tests/golden/ml_small.npz; 671 users x 9,066
  items, 100,004 ratings) repacked by ``tests/golden/make_golden.py`` into a
  compact ``.npz`` fixture, with ids numbered by sorted unique id the way the
  reference's ``Vocabulary`` does for ``from_interactions_df`` input
  (SURVEY.md §8d, config 1).
* ``synth_interactions()`` — the ML-25M-shaped synthetic generator specified in
  SURVEY.md §8(d) (configs 2-5).

``InteractionCSR`` is the minimal host container that plays the role of the
reference's ``SparseRowArray`` (``src/lenskit/data/matrix.py:318-540``): int32
(or int64) offsets, int32 sorted column indices, float32 values, kept as three
separate contiguous arrays exactly as the Arrow ``List<Struct{index,value}>``
storage does (struct children are separate buffers).
"""

from __future__ import annotations

from dataclasses import dataclass
from pathlib import Path

import numpy as np
import scipy.sparse as sps

GOLDEN_DIR = Path(__file__).resolve().parent.parent / "tests" / "golden"

#: approximate ML-25M rating histogram for values 0.5, 1.0, ..., 5.0 (SURVEY.md §8d)
ML_RATING_PMF = np.array(
    [0.016, 0.031, 0.016, 0.066, 0.050, 0.196, 0.127, 0.266, 0.088, 0.144], dtype=np.float64
)
ML_RATING_VALUES = np.arange(1, 11, dtype=np.float32) * np.float32(0.5)

ML25M_SHAPE = dict(n_users=162_541, n_items=59_047, nnz=25_000_095, seed=20260924)


@dataclass
class InteractionCSR:
    """Host CSR matrix (the ``SparseRowArray`` stand-in)."""

    indptr: np.ndarray  # int32 [n_rows+1] (int64 when nnz >= 2**31)
    indices: np.ndarray  # int32 [nnz], sorted within each row
    values: np.ndarray  # float32 [nnz]
    shape: tuple[int, int]

    @classmethod
    def from_scipy(cls, mat) -> "InteractionCSR":
        """Mirror of ``SparseRowArray.from_scipy`` (matrix.py:388-424)."""
        csr = sps.csr_array(mat)
        csr.sort_indices()
        smax = np.iinfo(np.int32).max
        odt = np.int32 if csr.nnz < smax else np.int64
        return cls(
            np.require(csr.indptr, dtype=odt, requirements="C"),
            np.require(csr.indices, dtype=np.int32, requirements="C"),
            np.require(csr.data, dtype=np.float32, requirements="C"),
            (int(csr.shape[0]), int(csr.shape[1])),
        )

    def to_scipy(self) -> sps.csr_array:
        return sps.csr_array((self.values, self.indices, self.indptr), shape=self.shape)

    @property
    def nnz(self) -> int:
        return int(self.indptr[-1])

    def __len__(self) -> int:
        return self.shape[0]


@dataclass
class Interactions:
    """COO interactions with numbered users/items (sorted, deduplicated)."""

    users: np.ndarray  # int32 [nnz]
    items: np.ndarray  # int32 [nnz]
    ratings: np.ndarray  # float32 [nnz]
    n_users: int
    n_items: int
    user_ids: np.ndarray | None = None  # original ids (ml-small only)
    item_ids: np.ndarray | None = None

    @property
    def nnz(self) -> int:
        return len(self.users)

    def coo(self, values: np.ndarray | None = None) -> sps.coo_array:
        v = self.ratings if values is None else values
        return sps.coo_array((v, (self.users, self.items)), shape=(self.n_users, self.n_items))


def synth_interactions_cached(path: str | None, **shape) -> Interactions:
    """``synth_interactions(**shape)`` through an optional ``.npz`` file: profiling scripts run the benchmark
    several times on one box and the generator takes half a minute; the cached arrays are the generator's own
    (same seed, same bits)."""
    import os

    if not path:
        return synth_interactions(**shape)
    key = np.array([shape["n_users"], shape["n_items"], shape["nnz"], shape.get("seed", 20260924)], dtype=np.int64)
    if os.path.exists(path):
        z = np.load(path)
        if np.array_equal(z["key"], key):
            return Interactions(z["users"], z["items"], z["ratings"], int(key[0]), int(key[1]))
    inter = synth_interactions(**shape)
    tmp = f"{path}.{os.getpid()}.tmp.npz"
    np.savez(tmp, key=key, users=inter.users, items=inter.items, ratings=inter.ratings)
    os.replace(tmp, path)
    return inter


def load_ml_small() -> Interactions:
    """Load the ml-latest-small fixture (see module docstring)."""
    f = GOLDEN_DIR / "ml_small.npz"
    z = np.load(f)
    user_ids = z["user_ids"]
    item_ids = z["item_ids"]
    return Interactions(
        users=z["users"].astype(np.int32),
        items=z["items"].astype(np.int32),
        ratings=(z["rating_halves"].astype(np.float32) * np.float32(0.5)),
        n_users=len(user_ids),
        n_items=len(item_ids),
        user_ids=user_ids,
        item_ids=item_ids,
    )


def synth_interactions(
    n_users: int, n_items: int, nnz: int, seed: int = 20260924, *, ratings: bool = True
) -> Interactions:
    """
    ML-25M-shaped synthetic interactions (SURVEY.md §8d).

    User weights LogNormal(0, 1.25), item weights (rank+20)^-1.05 with the
    rank->item-id map a seeded permutation; ceil(1.25*nnz) i.i.d. pairs are
    drawn, de-duplicated, shuffled, cut to ``nnz`` and sorted by (user, item).
    RNG draw order: user weights, permutation, users, items, shuffle, ratings.
    """
    rng = np.random.default_rng(seed)
    uw = rng.lognormal(0.0, 1.25, size=n_users)
    uw /= uw.sum()
    iw = (np.arange(n_items, dtype=np.float64) + 20.0) ** -1.05
    iw /= iw.sum()
    perm = rng.permutation(n_items)

    want = int(np.ceil(1.25 * nnz))
    max_pairs = n_users * n_items
    if nnz > max_pairs:
        raise ValueError("nnz exceeds matrix capacity")
    ucdf = np.cumsum(uw)
    icdf = np.cumsum(iw)
    ucdf[-1] = 1.0
    icdf[-1] = 1.0
    keys = np.empty(0, dtype=np.int64)
    # a couple of top-up rounds cover the duplicates lost on small dense shapes
    for _round in range(8):
        us = np.searchsorted(ucdf, rng.random(want), side="right").astype(np.int64)
        ranks = np.searchsorted(icdf, rng.random(want), side="right")
        its = perm[ranks].astype(np.int64)
        new = np.sort(us * n_items + its)  # np.unique is far slower than sort + mask here
        if len(keys):
            new = np.sort(np.concatenate([keys, new]))
        keys = new[np.concatenate([[True], new[1:] != new[:-1]])] if len(new) else new
        if len(keys) >= nnz:
            break
    if len(keys) < nnz:
        raise ValueError(f"could only draw {len(keys)} distinct pairs of {nnz}")
    rng.shuffle(keys)
    keys = np.sort(keys[:nnz])
    users = (keys // n_items).astype(np.int32)
    items = (keys % n_items).astype(np.int32)
    if ratings:
        pmf = ML_RATING_PMF / ML_RATING_PMF.sum()
        rv = ML_RATING_VALUES[rng.choice(len(pmf), size=nnz, p=pmf)]
    else:
        rv = np.ones(nnz, dtype=np.float32)
    return Interactions(users, items, rv.astype(np.float32), n_users, n_items)


def als_implicit_matrices(
    inter: Interactions, weight: float = 40.0, use_ratings: bool = False
) -> tuple[InteractionCSR, InteractionCSR]:
    """
    Build ``ui_rates`` / ``iu_rates`` the way ``ImplicitMFTrainer.prepare_matrix``
    and ``ALSTrainerBase.__init__`` do (``als/_implicit.py:141-149``,
    ``als/_common.py:216-219``): values = (1 or rating) * weight as f32.
    """
    base = inter.ratings if use_ratings else np.ones(inter.nnz, dtype=np.float32)
    vals = np.require(base, dtype=np.float32) * weight
    vals = vals.astype(np.float32)
    coo = inter.coo(vals)
    return InteractionCSR.from_scipy(coo), InteractionCSR.from_scipy(coo.T)


def knn_item_matrices(
    inter: Interactions, explicit: bool = True
) -> tuple[InteractionCSR, InteractionCSR, np.ndarray | None]:
    """
    Host prep of ``ItemKNNScorer.train`` (``knn/item.py:141-157,202-228``):
    per-item mean-centring (explicit only; f32 means) and unit-L2 normalisation
    of item columns with **f64** norms / reciprocal, cast to f32.  Uses the same
    SciPy calls as the reference so the f32 inputs are bit-identical
    (SURVEY.md Appendix B).  Returns (UI, IU, item_means).
    """
    import scipy.sparse.linalg as spla

    vals = inter.ratings if explicit else np.ones(inter.nnz, dtype=np.float32)
    rmat = inter.coo(vals.astype(np.float32)).astype(np.float32)
    means = None
    if explicit:
        rmat = rmat.tocsc()
        counts = np.diff(rmat.indptr)
        sums = rmat.sum(axis=0)
        means = np.zeros(sums.shape, dtype=np.float32)
        np.divide(sums, counts, out=means, where=counts > 0)
        rmat.data = rmat.data - np.repeat(means, counts)
        if np.allclose(rmat.data, 0.0):  # checked on the centred values, before normalisation (knn/item.py:211-216)
            import warnings

            warnings.warn("Ratings seem to have the same value, centering is not recommended.", UserWarning)
    norms = spla.norm(rmat, 2, axis=0)
    cmat = rmat / np.maximum(norms, np.finfo("f4").smallest_normal)
    cmat = cmat.astype(np.float32)
    ui = InteractionCSR.from_scipy(cmat.tocsr())
    iu = InteractionCSR.from_scipy(cmat.T.tocsr())
    return ui, iu, (None if means is None else np.asarray(means))
