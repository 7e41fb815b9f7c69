"""
Association and SLIM scoring, and association training, on catalogues wider than one column tile ("half") of
``lk_assoc_score_batch`` / ``lk_cooc_count``, bit for bit against ``tests/cooc_oracle.py``, ``tests/slim_oracle.py``
and ``oracle.argtopn``.

The shapes come from ``lk_cooc_geometry``: the smallest item count with two halves (its last half holds one item),
one in the middle of the two-half range, and the ML-25M item count.  Every test asserts its number of halves, so a
change of the tiling cannot quietly turn it back into a one-half test.  Only the item count is large; the matrices
and the interaction data are small.
"""

import ctypes as C
import functools

import numpy as np
import pyarrow as pa
import pytest
import torch

import cooc_oracle as co
import oracle
import slim_oracle as so
from lkpy_b200 import _lib, accel, data, engine
from lkpy_b200.association import AssociationScorer
from lkpy_b200.components import Dataset, ItemList
from lkpy_b200.slim import SLIMScorer

pytestmark = pytest.mark.gpu

ML25M_ITEMS = data.ML25M_SHAPE["n_items"]


def _geom(n_items: int) -> engine.LkKnnGeom:
    g = engine.LkKnnGeom()
    _lib.check(_lib.lib().lk_cooc_geometry(n_items, n_items, C.byref(g)), "lk_cooc_geometry")
    return g


@functools.cache
def _first_with(halves: int) -> int:
    """The smallest item count the geometry splits into ``halves`` column tiles (n_halves never decreases with n)."""
    lo, hi = 1, 1 << 24
    assert _geom(hi).n_halves >= halves
    while lo < hi:
        mid = (lo + hi) // 2
        if _geom(mid).n_halves >= halves:
            hi = mid
        else:
            lo = mid + 1
    return lo


def _shape(which: str) -> int:
    two = _first_with(2)
    if which == "two_min":
        return two
    if which == "two_mid":
        return (two + _first_with(3)) // 2
    return ML25M_ITEMS


SHAPES = ["two_min", "two_mid", "ml25m"]


def _tiling(n: int):
    """(tile_cols, columns per half, halves) of an n-item association matrix, checked to span several halves."""
    g = _geom(n)
    TW, CW, H = g.tile_cols, g.warps * g.tile_cols, g.n_halves
    assert H >= 2 and (H - 1) * CW < n <= H * CW
    if n == ML25M_ITEMS:
        assert H == 3
    if n == _first_with(2):
        assert n - CW == 1  # the last half holds a single item
    return TW, CW, H


def _boundaries(n: int) -> np.ndarray:
    TW, CW, _H = _tiling(n)
    b = np.array([0, TW - 1, TW, CW - 1, CW, CW + 1, 2 * CW - 1, 2 * CW, n - 1])
    return np.unique(b[b < n])


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_lib.require_device())


def _ragged(lists):
    ptr = np.zeros(len(lists) + 1, np.int64)
    ptr[1:] = np.cumsum([len(x) for x in lists])
    items = np.concatenate(lists).astype(np.int32) if lists else np.zeros(0, np.int32)
    return ptr, items


def _csr(n: int, rows: dict) -> tuple:
    """Host CSR (int64 offsets, columns ascending) of ``{row: (cols, vals)}``; other rows are empty."""
    lens = np.zeros(n, np.int64)
    for r, (c, _v) in rows.items():
        lens[r] = len(c)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    cols = np.zeros(int(indptr[-1]), np.int32)
    vals = np.zeros(int(indptr[-1]), np.float32)
    for r, (c, v) in rows.items():
        o = np.argsort(c, kind="stable")
        cols[indptr[r] : indptr[r + 1]] = np.asarray(c)[o]
        vals[indptr[r] : indptr[r + 1]] = np.asarray(v, np.float32)[o]
    return indptr, cols, vals


def _check_tile_ptr(st: engine.AssocState):
    """tile_ptr[r, s] = searchsorted(row r's columns, s * tile_cols) - row start, for every row and subtile."""
    g = st.geom
    S1 = g.n_subtiles + 1
    indptr = st.indptr.cpu().numpy()
    nnz = int(indptr[-1])
    cols = st.cols.cpu().numpy()[:nnz].astype(np.int64)
    n = st.n_items
    got = st.tile_ptr.cpu().numpy()[: n * S1].reshape(n, S1)
    row = np.repeat(np.arange(n), np.diff(indptr))
    want = np.zeros((n, S1), np.int64)
    for s in range(S1):
        want[:, s] = np.bincount(row[cols < s * g.tile_cols], minlength=n)  # = searchsorted in an ascending row
    for r in np.flatnonzero(np.diff(indptr))[:16]:  # spelled out on a few rows
        rc = cols[indptr[r] : indptr[r + 1]]
        assert np.array_equal(want[r], np.searchsorted(rc, np.arange(S1) * g.tile_cols)), r
    assert np.array_equal(got, want)


# ---------------------------------------------------------------------------
# the kernel on a hand-built matrix
# ---------------------------------------------------------------------------


def _synth_matrix(n: int, seed: int = 0):
    """
    A matrix whose rows hit the half boundaries: ``roles`` maps a role to its row number(s).  Values are multiples of
    1/4 in [-2, 2] (agg 0 and 2; the non-negative matrix, |v|, for agg 1), so that many scores tie.
    """
    TW, CW, H = _tiling(n)
    bnd = _boundaries(n)
    rng = np.random.default_rng(seed)
    # row numbers at the boundaries too: the tile pointers of the last row and of the first row of a half
    span = [0, int(CW), int(n - 1), 5, int(CW - 1)]
    roles = dict(span=span, last=int(TW), sparse=int(CW + 1) if CW + 1 < n else 7, empty=int(TW - 1))
    rows = {}
    for k, r in enumerate(span):
        c = np.unique(np.concatenate([bnd if k % 2 == 0 else bnd[::2], rng.integers(0, n, 300)]))
        rows[r] = (c, rng.integers(-8, 9, len(c)) * 0.25)
    last = np.unique(np.concatenate([[n - 1], rng.integers((H - 1) * CW, n, 40)]))
    rows[roles["last"]] = (last, rng.integers(1, 9, len(last)) * 0.25)
    # few non-zero scores, none in half 0: its zeros fill the heap there and must be evicted in later halves
    few = np.unique([(H - 1) * CW, n - 1, CW, CW + 1 if CW + 1 < n else CW])
    rows[roles["sparse"]] = (few, np.full(len(few), 0.5))
    assert roles["empty"] not in rows
    ip, cols, vals = _csr(n, rows)
    return roles, ip, cols, vals


def _synth_queries(roles):
    s, last, sparse, empty = roles["span"], roles["last"], roles["sparse"], roles["empty"]
    return [
        np.array([last]),  # every entry in the last half
        np.array(s[:3]),  # rows spanning all halves
        np.array([s[0], s[3], s[0], last, s[3], s[1]]),  # repeated reference items
        np.zeros(0, np.int64),  # no reference items
        np.array([sparse]),  # fewer non-zero scores than n
        np.array([empty]),  # an empty reference row: every score 0
        np.array(s + [empty, last]),  # every kind of row; its exclusions cover all of half 0
        np.array([s[4], s[2]]),
    ]


def _synth_exclusions(n: int, B: int, seed: int = 1):
    """Unsorted lists with repeats, negative and unknown numbers, items in every half and the boundary columns;
    query 6 excludes every item of half 0."""
    _TW, CW, H = _tiling(n)
    bnd = _boundaries(n)
    rng = np.random.default_rng(seed)
    lists = []
    for b in range(B):
        kind = b % 4
        if b == 6:
            e = np.concatenate([rng.permutation(CW), [-1, CW - 1, 0]])
        elif kind == 0:
            e = np.zeros(0, np.int64)
        elif kind == 1:
            e = np.concatenate([rng.permutation(bnd), bnd[:3], rng.integers(0, n, 30)])
        elif kind == 2:
            e = np.concatenate([[-1, -7], rng.integers((H - 1) * CW, n, 10), [-1], bnd[-2:], [n + 3]])
        else:
            e = np.concatenate([rng.integers(h * CW, min((h + 1) * CW, n), 8) for h in range(H)] + [bnd, [-2]])
        lists.append(np.asarray(e, dtype=np.int32))
    return lists


def _dense(st_host, refs):
    return st_host[np.asarray(refs, np.int64), :].toarray().astype(np.float32)


def _restated(st_host, refs, agg: int) -> np.ndarray:
    """The kernel's scores in f32 sequential order: the mean (score_sequential), the sum, the max from +0.0."""
    n = st_host.shape[1]
    if len(refs) == 0:
        return np.zeros(n, np.float32) if agg == 2 else np.full(n, np.nan, np.float32)
    rows = _dense(st_host, refs)
    with np.errstate(invalid="ignore"):
        if agg == 0:
            return co.score_sequential(rows)
        s = np.zeros(n, np.float32)
        for row in rows:
            s = s + row if agg == 2 else np.maximum(s, row)
        return s


def _check_scores(got, want):
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    assert np.array_equal(_bits(got[ok]), _bits(want[ok]))


def _check_rank(idx, val, cnt, S, n, lists=None):
    for b, s in enumerate(S):
        col = s.copy()
        if lists is not None:
            e = lists[b]
            col[e[(e >= 0) & (e < len(col))]] = np.nan
        want = oracle.argtopn(col, n)
        c = int(cnt[b])
        assert c == len(want) == min(n, int((~np.isnan(col)).sum())), (b, n)
        assert np.array_equal(idx[b, :c], want), (b, n)
        assert np.array_equal(_bits(val[b, :c]), _bits(col[want])), (b, n)
        assert np.all(idx[b, c:] == -1) and np.all(np.isnan(val[b, c:])), (b, n)


def _state(n, ip, cols, vals):
    st = engine.AssocState.create(n, ip, cols, vals)
    _check_tile_ptr(st)
    return st


@pytest.mark.parametrize("agg", [0, 1, 2])
@pytest.mark.parametrize("which", SHAPES)
def test_kernel_across_halves(cuda_lib, which, agg):
    n = _shape(which)
    roles, ip, cols, vals = _synth_matrix(n)
    if agg == 1:  # the max starts at +0.0: the matrix must be non-negative, as training makes it
        vals = np.abs(vals)
    st = _state(n, ip, cols, vals)
    host = st.host_csr()
    qs = _synth_queries(roles)
    r_ptr, r_items = _ragged(qs)
    r_ptr, r_items = _t(r_ptr), _t(r_items)
    S = np.stack([_restated(host, q, agg) for q in qs])

    got = st.score(r_ptr, r_items, agg).cpu().numpy()
    for b in range(len(qs)):
        _check_scores(got[b], S[b])

    lists = _synth_exclusions(n, len(qs))
    e_ptr, e_items = _ragged(lists)
    for nn in (1, 10, 100, 1024):
        for excl in (None, lists):
            ex = (_t(e_ptr), _t(e_items)) if excl is not None else (None, None)
            idx, val, cnt = (t.cpu().numpy() for t in st.recommend(r_ptr, r_items, agg, nn, *ex))
            _check_rank(idx, val, cnt, S, nn, excl)


def test_nan_scores_are_never_offered(cuda_lib):
    """+inf and -inf at one column of two reference rows make a NaN mean and sum there; item 0 is the first
    offer.  Rank mode skips NaN scores as argtopn does."""
    n = ML25M_ITEMS
    _TW, CW, _H = _tiling(n)
    bnd = _boundaries(n)
    nan_at = np.array([0, CW, n - 1])
    rng = np.random.default_rng(4)
    rows = {}
    for r, sign in ((3, 1.0), (CW + 2, -1.0)):
        c = np.unique(np.concatenate([bnd, rng.integers(0, n, 200)]))
        v = rng.integers(-8, 9, len(c)) * 0.25
        v[np.isin(c, nan_at)] = sign * np.inf
        rows[r] = (c, v)
    c = np.unique(rng.integers(0, n, 50))
    rows[n - 2] = (c, np.full(len(c), 0.75))
    st = _state(n, *_csr(n, rows))
    host = st.host_csr()
    qs = [np.array([3, CW + 2]), np.array([CW + 2, n - 2, 3]), np.array([3])]
    r_ptr, r_items = (_t(a) for a in _ragged(qs))
    lists = _synth_exclusions(n, len(qs))
    e_ptr, e_items = _ragged(lists)
    for agg in (0, 2):
        S = np.stack([_restated(host, q, agg) for q in qs])
        assert np.array_equal(np.flatnonzero(np.isnan(S[0])), nan_at)
        assert np.array_equal(np.flatnonzero(np.isnan(S[1])), nan_at)
        got = st.score(r_ptr, r_items, agg).cpu().numpy()
        for b in range(len(qs)):
            _check_scores(got[b], S[b])
        for nn in (1, 10, 100, 1024):
            for excl in (None, lists):
                ex = (_t(e_ptr), _t(e_items)) if excl is not None else (None, None)
                idx, val, cnt = (t.cpu().numpy() for t in st.recommend(r_ptr, r_items, agg, nn, *ex))
                _check_rank(idx, val, cnt, S, nn, excl)


# ---------------------------------------------------------------------------
# training and the scorers on a dataset wider than one half
# ---------------------------------------------------------------------------


def _with_users(it: data.Interactions, extra: list) -> data.Interactions:
    """``it`` with the item lists ``extra`` appended as new users (sorted, de-duplicated)."""
    u = np.concatenate([it.users] + [np.full(len(x), it.n_users + k) for k, x in enumerate(extra)]).astype(np.int64)
    i = np.concatenate([it.items] + [np.asarray(x) for x in extra]).astype(np.int64)
    keys = np.unique(u * it.n_items + i)
    return data.Interactions((keys // it.n_items).astype(np.int32), (keys % it.n_items).astype(np.int32),
                             np.ones(len(keys), np.float32), it.n_users + len(extra), it.n_items)  # fmt: skip


@pytest.fixture(scope="module")
def wide():
    """ML-25M's item count, few users: the synthetic interactions plus users holding the boundary columns (three
    alike, so that SLIM's weights there pass the L1 threshold) and one whose items all lie in the last half."""
    n = ML25M_ITEMS
    _TW, CW, H = _tiling(n)
    bnd = _boundaries(n)
    it = data.synth_interactions(600, n, 20_000, seed=11)
    last = np.random.default_rng(5).integers((H - 1) * CW, n, 30)
    it = _with_users(it, [bnd, bnd, bnd, np.concatenate([bnd[::2], [17, 40_000]]), last])
    hand = np.arange(it.n_users - 5, it.n_users)
    assert np.all(np.bincount(it.items // CW, minlength=H) > 100)
    return Dataset(it), hand


def _dup_groups(n: int, seed=3, n_groups=300, nnz=20_000):
    """Groups ascending, repeats inside groups, an empty group; zipf items spread over every half by a
    permutation, and three groups with repeated boundary columns."""
    rng = np.random.default_rng(seed)
    perm = rng.permutation(n)
    g = np.sort(rng.integers(0, n_groups, nnz))
    i = perm[rng.zipf(1.3, nnz) % (n - 5)]
    g[g == 7] = 8
    bnd = _boundaries(n)
    extra = [np.concatenate([bnd, bnd[::-1], bnd[:2]]), bnd, rng.permutation(np.repeat(bnd, 3))]
    g = np.concatenate([g] + [np.full(len(x), n_groups + k) for k, x in enumerate(extra)])
    i = np.concatenate([i] + extra)
    return n_groups + len(extra), g.astype(np.int32), i.astype(np.int32)


@pytest.mark.parametrize("which", ["wide", "dups"])
def test_count_cooc(cuda_lib, wide, which):
    if which == "wide":
        it = wide[0].interactions
        ng, ni, g, i = it.n_users, it.n_items, it.users, it.items
    else:
        ni = _shape("two_mid")
        ng, g, i = _dup_groups(ni)
    _tiling(ni)
    got = accel.run_accel_task(accel.data.count_cooc(ng, ni, pa.array(g), pa.array(i)))
    want = co.count_cooc(ng, ni, g, i)
    assert len(got) == len(want)
    for b, w in zip(got, want):
        for k, col in enumerate(("row", "col", "count")):
            assert np.array_equal(b.column(col).to_numpy(), w[k]), col
    _TW, CW, H = _tiling(ni)
    assert np.any(want[1][1] >= (H - 1) * CW)  # counts in the last half's columns


CONFIGS = [dict(method="probability"), dict(method="lift"), dict(method="lift", damping=0.1)]


@pytest.fixture(scope="module", params=range(len(CONFIGS)), ids=["probability", "lift", "lift_damped"])
def trained(request, wide):
    ds, _hand = wide
    cfg = CONFIGS[request.param]
    m = AssociationScorer(**cfg)
    m.train(ds)
    return cfg, m


def _wide_queries(ds, hand, rng, n=20):
    it = ds.interactions
    qs = []
    for u in list(rng.choice(it.n_users - len(hand), n, replace=False)) + list(hand):
        nums = ds.user_history(int(u)).numbers()
        if u % 3 == 0:  # repeated reference items
            nums = np.concatenate([nums, nums[: max(1, len(nums) // 3)]])
        qs.append(rng.permutation(nums) if u % 2 else nums)
    qs.append(np.zeros(0, np.int32))
    return qs


def test_assoc_train_and_score(cuda_lib, wide, trained):
    ds, hand = wide
    cfg, m = trained
    it = ds.interactions
    st = m._device_state()
    _check_tile_ptr(st)
    want = co.assoc_matrix(it.n_users, it.n_items, it.users, it.items, cfg["method"], cfg.get("damping", 0.0))
    A = m.assoc_scores
    assert np.array_equal(A.indptr, want.indptr) and np.array_equal(A.indices, want.indices)
    assert np.array_equal(_bits(A.data), _bits(want.data))
    _TW, CW, H = _tiling(it.n_items)
    assert np.any(A.indices >= (H - 1) * CW)

    rng = np.random.default_rng(1)
    qs = _wide_queries(ds, hand, rng)
    hist = [ItemList(item_nums=q, vocabulary=ds.items) for q in qs]
    tgt_nums = np.concatenate([_boundaries(it.n_items), rng.integers(0, it.n_items, 500)])
    tgt = ItemList(item_nums=tgt_nums, vocabulary=ds.items)
    for max_nbrs in (None, 1):
        m.config = m.config.model_copy(update={"max_nbrs": max_nbrs})
        got = m.score_batch(hist, [tgt] * len(hist))
        for q, g in zip(qs, got):
            _check_scores(g.scores(), co.score(A, q, max_nbrs)[tgt_nums])
    m.config = m.config.model_copy(update={"max_nbrs": None})


@pytest.mark.parametrize("exclude", ["query", None])
@pytest.mark.parametrize("max_nbrs", [None, 1])
def test_assoc_recommend(cuda_lib, wide, exclude, max_nbrs):
    ds, hand = wide
    m = AssociationScorer(method="lift", damping=0.1, max_nbrs=max_nbrs)
    m.train(ds)
    A = m.assoc_scores
    rng = np.random.default_rng(2)
    qs = _wide_queries(ds, hand, rng, 15)
    qs.append(ds.user_history(int(hand[-1])).numbers()[:1])  # one reference row, in the last half
    qs.append(np.array([int(np.argmin(np.diff(A.indptr)))], np.int32))  # few non-zero scores: zero ties fill lists
    hist = [ItemList(item_nums=q, vocabulary=ds.items) for q in qs]
    for n in (1, 10, 1024):
        got = m.recommend_batch(hist, n, exclude=exclude)
        for q, g in zip(qs, got):
            s = co.score(A, q, max_nbrs).copy()
            if exclude == "query":
                s[q] = np.nan
            want = oracle.argtopn(s, n)
            assert np.array_equal(g.numbers(), want)
            assert np.array_equal(_bits(g.scores()), _bits(s[want]))


@pytest.fixture(scope="module")
def slim(wide):
    ds, _hand = wide
    m = SLIMScorer(max_nbrs=20)
    m.train(ds)
    return m


def test_slim_train_and_score(cuda_lib, wide, slim):
    ds, hand = wide
    it = ds.interactions
    ui = so.structure(it.n_users, it.users, it.items)
    iu = so.structure(it.n_items, it.items, it.users)
    want = so.train(it.n_users, it.n_items, ui, iu, 1.0, 1.0, 100, 20).T.tocsr()
    W = slim.weights
    assert np.array_equal(W.indptr, want.indptr) and np.array_equal(W.indices, want.indices)
    assert np.array_equal(_bits(W.data), _bits(want.data))
    _TW, CW, H = _tiling(it.n_items)
    assert np.any(W.indices >= (H - 1) * CW) and np.any(np.diff(W.indptr)[(H - 1) * CW :])
    _check_tile_ptr(slim._device_state())

    rng = np.random.default_rng(3)
    qs = _wide_queries(ds, hand, rng)
    hist = [ItemList(item_nums=q, vocabulary=ds.items) for q in qs]
    tgt_nums = np.concatenate([_boundaries(it.n_items), rng.integers(0, it.n_items, 500)])
    tgt = ItemList(item_nums=tgt_nums, vocabulary=ds.items)
    for q, g in zip(qs, slim.score_batch(hist, [tgt] * len(hist))):
        s = g.scores()
        if len(q):
            _check_scores(s, so.score(W, q)[tgt_nums])
        else:
            assert np.all(np.isnan(s))
    for n in (1, 10, 1024):
        for exclude in ("query", None):
            recs = slim.recommend_batch(hist, n, exclude=exclude)
            for q, rec in zip(qs, recs):
                if not len(q):
                    assert len(rec) == 0
                    continue
                s = so.score(W, q)
                if exclude == "query":
                    s[q] = np.nan
                want = oracle.argtopn(s, n)
                assert np.array_equal(rec.numbers(), want), n
                assert np.array_equal(_bits(rec.scores()), _bits(s[want]))
