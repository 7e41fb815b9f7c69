"""
The reference's own ``stochastic/_ranker.py`` (``StochasticTopNRanker``) and ``random.py`` on top of the sandbox of
``ref_sandbox``; and the recording of its calls that ``tests/golden/reference_classes/stochastic_*.npz`` holds.

``ItemList.top_n`` reaches ``_accel.data.argtopn``, the reference's Rust heap; here that is the heap replay of
tests/stochastic_oracle.py over the f64 keys (``ref_sandbox``'s stand-in is this package's f32 kernel).  Everything
else, from the configuration to the keys, is the reference's code.
"""

from __future__ import annotations

import contextlib
import sys

import numpy as np

import ref_sandbox
import stochastic_oracle as so

#: the recorded configurations, by golden-file name
CASES = {
    "stochastic_softmax": {"rng": 1234, "transform": "softmax"},
    "stochastic_softmax_overflow": {"rng": 77, "transform": "softmax", "scale": 1e4, "n": 8},
    "stochastic_linear": {"rng": 5, "transform": "linear", "scale": 0.1},
    "stochastic_none": {"rng": 9, "transform": None, "n": 12},
    "stochastic_user_int": {"rng": (99, "user"), "transform": "softmax"},
    "stochastic_user_str": {"rng": (31, "user"), "transform": "linear", "scale": 1e4},
}
#: the ``n`` of each call (None: the call passes none)
CALL_N = [10, None, 0, 3, -1, 500, 1, 25]
NONE_N = -999


def calls(name: str):
    """``(scores, user id or None, n, include_weights)`` of every recorded call of case ``name``: lists with NaN,
    ±inf and ties, an empty and an all-invalid list, int, str and missing user ids."""
    rng = np.random.default_rng(sum(map(ord, name)))
    out = []
    for c, n in enumerate(CALL_N):
        L = int(rng.integers(5, 60))
        s = rng.standard_normal(L).astype(np.float32) * np.float32(2.0)
        if c % 3 == 1:
            s = (np.round(s * 2) / 2).astype(np.float32)  # ties among the scores
        bad = rng.random(L)
        s[bad < 0.1] = np.nan
        s[(bad >= 0.1) & (bad < 0.14)] = np.inf
        s[(bad >= 0.14) & (bad < 0.17)] = -np.inf
        if c == 6:
            s = np.zeros(0, np.float32)
        elif c == 7:
            s[:] = np.nan
        user = None
        if name.startswith("stochastic_user") and c % 4 != 2:
            user = int(rng.integers(1, 1000)) if name.endswith("int") else f"u{int(rng.integers(1, 1000))}"
        out.append((s, user, n, c != 3))
    return out


@contextlib.contextmanager
def stochastic_modules():
    """``ref_sandbox.reference_modules()`` plus ``stochastic/_ranker.py``, with argtopn over f64 keys."""
    import pyarrow as pa

    with ref_sandbox.reference_modules() as mods:
        ref_sandbox._module("lenskit.stochastic", package=True)
        sys.modules["lenskit._accel"].data.argtopn = lambda scores, n: pa.array(
            so.argtopn(np.asarray(scores.to_numpy(zero_copy_only=False), np.float64), n), type=pa.int32()
        )
        mods["lenskit.stochastic._ranker"] = ref_sandbox._load("lenskit.stochastic._ranker", "stochastic/_ranker.py")
        yield mods


def record() -> dict[str, dict]:
    """Every case's calls through the reference class: the lists, the picked positions and their keys, and for a
    fixed generator its PCG64 state afterwards.  Adjacent recorded keys differ by at least 1e-5 relative, so that the
    order they give holds within the tolerance the keys are compared with."""
    out = {}
    with stochastic_modules() as ref:
        rk, ItemList = ref["lenskit.stochastic._ranker"], ref["lenskit.data._items"].ItemList
        for name, cfg in CASES.items():
            r = rk.StochasticTopNRanker(rk.StochasticTopNConfig(**cfg))
            cs = calls(name)
            Lmax = max(len(s) for s, *_ in cs)
            scores = np.full((len(cs), Lmax), np.nan, np.float32)
            pos, keys, ptr = [], [], [0]
            for c, (s, user, n, weights) in enumerate(cs):
                scores[c, : len(s)] = s
                res = r(ItemList(item_ids=np.arange(len(s)), scores=s), user, n, include_weights=weights)
                p = np.asarray(res.ids(), np.int64)
                w = res.field("weight") if weights else None  # a list with nothing valid returns without one
                k = np.full(len(p), np.nan) if w is None else np.asarray(w, np.float64)
                if weights and len(k) > 1:
                    gap = np.abs(np.diff(k)) / np.abs(k[1:])
                    assert gap.min() >= 1e-5, (name, c, gap.min())
                pos.append(p)
                keys.append(k)
                ptr.append(ptr[-1] + len(p))
            d = {
                "scores": scores, "lens": np.array([len(s) for s, *_ in cs]),
                "users": np.array(["" if u is None else str(u) for _s, u, *_ in cs]),
                "user_kind": np.array([0 if u is None else (1 if isinstance(u, int) else 2) for _s, u, *_ in cs]),
                "n": np.array([NONE_N if n is None else n for _s, _u, n, _w in cs]),
                "weights": np.array([w for *_, w in cs]),
                "ptr": np.array(ptr), "pos": np.concatenate(pos), "keys": np.concatenate(keys),
            }  # fmt: skip
            f = r._rng_factory
            if hasattr(f, "rng"):
                st = f.rng.bit_generator.state["state"]
                d["state"] = np.array([st["state"] >> 64, st["state"] % 2**64, st["inc"] >> 64, st["inc"] % 2**64],
                                      np.uint64)  # fmt: skip
            out[name] = d
    return out
