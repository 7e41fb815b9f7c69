"""
Host restatements for the bias model and the offset scorers (tests/test_basic*.py):

* NumPy's pairwise f32 sum, and the global mean the way ``lk_bias_learn`` evaluates it — the tree cut at
  ``MEAN_DEPTH``, each subtree summed on its own, the inner nodes above combined level by level;
* ratings on which the order of the learner's entity chains shows in the f32 biases, and the count of biases a
  reversed chain changes;
* ``BiasModel.compute_for_items`` (basic/bias.py), statement for statement, for one query: the user bias of its rated
  items (the oracle of ``basic.BiasModel.user_bias_for_items``) and the scores;
* the host composition a batched ranking must reproduce: scores, exclusions as NaN, ``argtopn``.
"""

from __future__ import annotations

import numpy as np

import oracle

MEAN_DEPTH = 16  # basic.cu


def split(n: int) -> int:
    n2 = n // 2
    return n2 - n2 % 8


def pairwise(a: np.ndarray) -> np.float32:
    """NumPy's pairwise sum of an f32 array (numpy/_core/src/umath/loops_utils.h.src)."""
    n = len(a)
    if n < 8:
        res = np.float32(0.0)
        for x in a:
            res = np.float32(res + x)
        return res
    if n <= 128:
        r = a[:8].copy()
        i = 8
        for i in range(8, n - n % 8, 8):
            r += a[i : i + 8]
        i = n - n % 8
        res = np.float32(np.float32(np.float32(r[0] + r[1]) + np.float32(r[2] + r[3]))
                         + np.float32(np.float32(r[4] + r[5]) + np.float32(r[6] + r[7])))  # fmt: skip
        for x in a[i:]:
            res = np.float32(res + x)
        return res
    n2 = split(n)
    return np.float32(pairwise(a[:n2]) + pairwise(a[n2:]))


def mean_node(nnz: int, d: int, p: int):
    """basic.cu's ``mean_node``: ``(lo, n)`` of the node at depth d along path p, or None when it does not exist."""
    lo, n = 0, nnz
    for k in range(d):
        if n <= 128:
            return (lo, n) if p & ((1 << (d - k)) - 1) == 0 else None
        n2 = split(n)
        if (p >> (d - 1 - k)) & 1:
            lo, n = lo + n2, n - n2
        else:
            n = n2
    return lo, n


def kernel_mean(r: np.ndarray) -> np.float32:
    """The global mean as ``lk_bias_learn`` computes it: every subtree at depth ``MEAN_DEPTH`` (or leaf above it)
    summed into the slot of its leftmost descendant, then the inner nodes level by level, deepest first."""
    r = np.ascontiguousarray(r, dtype=np.float32)
    nnz = len(r)
    part = {}

    def visit(lo: int, n: int, d: int, p: int) -> None:
        if d == MEAN_DEPTH or n <= 128:
            part[p << (MEAN_DEPTH - d)] = pairwise(r[lo : lo + n])
            return
        n2 = split(n)
        visit(lo, n2, d + 1, 2 * p)
        visit(lo + n2, n - n2, d + 1, 2 * p + 1)

    visit(0, nnz, 0, 0)
    if nnz > 128:
        for d in range(MEAN_DEPTH - 1, -1, -1):
            for p in range(1 << d):
                node = mean_node(nnz, d, p)
                if node is None or node[1] <= 128:
                    continue
                s = p << (MEAN_DEPTH - d)
                part[s] = np.float32(part[s] + part[s + (1 << (MEAN_DEPTH - d - 1))])
    total = np.float32(np.float32(0.0) + part[0])  # np.add.reduce starts from the identity
    return np.float32(np.float64(total) / np.float64(nnz))


def cancelling_ratings(it, rng: np.random.Generator, big: float = 2.0**36) -> np.ndarray:
    """``it.ratings`` with ``+big`` and ``-big`` added along 4-cycles of the rating matrix, in f32: for every item
    with two raters (u, v) who also rated the most rated item H, ``+big`` at (u, i) and (v, H), ``-big`` at
    (v, i) and (u, H) (the pair is drawn with ``rng``).  Every item's and every user's additions sum to zero, so a
    bias stays small while the partial sums of its chain pass through +-big.  There an f64 add rounds the
    ratings' low bits, and which ratings are rounded depends on the order of the chain.  A cell that gets an
    addition holds a multiple of ``big`` exactly (the rating is lost in f32)."""
    H = int(np.argmax(np.bincount(it.items, minlength=it.n_items)))
    h_pos = np.full(it.n_users, -1, np.int64)
    on_h = np.flatnonzero(it.items == H)
    h_pos[it.users[on_h]] = on_h
    cand = np.flatnonzero((it.items != H) & (h_pos[it.users] >= 0))
    cand = cand[rng.permutation(len(cand))]
    cand = cand[np.argsort(it.items[cand], kind="stable")]  # each item's candidates in a random order
    first = np.flatnonzero(np.concatenate([[True], it.items[cand[1:]] != it.items[cand[:-1]]]))
    two = np.diff(np.append(first, len(cand))) >= 2
    a, b = cand[first[two]], cand[first[two] + 1]
    d = np.zeros(it.nnz)
    np.add.at(d, a, big)
    np.add.at(d, b, -big)
    np.add.at(d, h_pos[it.users[a]], -big)
    np.add.at(d, h_pos[it.users[b]], big)
    return (np.asarray(it.ratings, np.float64) + d).astype(np.float32)


def reversed_chain_changes(it, centered_dtype) -> tuple[int, int]:
    """How many f32 item biases and f32 user biases of ``BiasModel.learn`` (damping 0, both entities) change bits
    when each entity's ``np.add.at`` chain runs in reverse COO order: ``(items, users)``.  These are the values
    the tests compare, so a count above zero means that a pass adding that entity's values out of order gives
    other output on ``it``.  The user values of both orders are centred by the forward item biases, so the user
    count is the user pass's own."""
    c = it.ratings.astype(centered_dtype) - float(np.mean(it.ratings))
    changed, ib = [], None
    for idx, n in ((it.items, it.n_items), (it.users, it.n_users)):
        vals = c if ib is None else c - ib[it.items]
        counts = np.bincount(idx, minlength=n).astype(np.float64)
        biases = []
        for order in (slice(None), slice(None, None, -1)):
            sums = np.zeros(n)
            np.add.at(sums, idx[order], vals[order])
            out = np.zeros(n, dtype=np.float32)
            np.divide(sums, counts, out=out, where=counts > 0, casting="unsafe")
            biases.append(out)
        changed.append(int((biases[0].view(np.int32) != biases[1].view(np.int32)).sum()))
        ib = biases[0]
    return changed[0], changed[1]


def bias_scores(model, users, items, query, targets) -> np.ndarray:
    """``BiasScorer.__call__``: ``model.compute_for_items(targets, query.user_id, query.query_items)``'s scores,
    with the reference's statements on ``lkpy_b200.basic.BiasModel`` (``damping`` as ``(user, item)``)."""
    scores = np.full(len(targets), model.global_bias, dtype=np.float32)
    if model.item_biases is not None:
        idxes = targets.numbers(vocabulary=items, missing="negative")
        mask = idxes >= 0
        scores[mask] += model.item_biases[idxes[mask]]
    user_items = query.query_items
    ratings = None if user_items is None else user_items.field("rating")
    if model.user_biases is not None:
        if ratings is not None:
            scores += rated_user_bias(model, items, user_items)
        elif query.user_id is not None:
            uno = users.number(query.user_id, missing="none")
            if uno is not None:
                scores += model.user_biases[uno]
    return scores


def rated_user_bias(model, items, user_items):
    """``compute_for_items``' user bias from the rated items ``user_items`` (they have a ``rating`` field)."""
    uoff = user_items.field("rating") - model.global_bias
    if model.item_biases is not None:
        r_idxes = user_items.numbers(vocabulary=items, missing="negative")
        r_mask = r_idxes >= 0
        uoff[r_mask] -= model.item_biases[r_idxes[r_mask]]
    user_bias = np.sum(uoff) / (np.sum(np.isfinite(uoff)) + model.damping[0])
    if np.isnan(user_bias):
        user_bias = 0
    return user_bias


def ranked(scores: np.ndarray, excluded, n: int) -> tuple[np.ndarray, np.ndarray]:
    """``TopNRanker`` after the candidate selector: the excluded items' scores NaN, then ``argtopn``."""
    s = np.array(scores, dtype=np.float32)
    ex = np.asarray(excluded, dtype=np.int64)
    s[ex[ex >= 0]] = np.nan
    idx = oracle.argtopn(s, n)
    return idx, s[idx]
