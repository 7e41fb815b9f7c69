"""
Plain restatements of the FlexMF implicit training pieces, for the tests and ``smoke()``:

* ``draw`` / ``sample_negatives``: the counter-based generator and the accept/reject loop that
  ``include/lkpy_b200.h`` defines for ``lk_flexmf_sample_negatives``, in NumPy;
* ``Model`` / ``train_step``: one minibatch step in plain torch on the CPU — embedding lookups, the logistic or
  pairwise loss, the L2 term, ``backward()`` and ``torch.optim.AdamW`` / ``SparseAdam`` — parameterised on dtype.
"""

from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

_M1, _M2, _G = np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB), np.uint64(0x9E3779B97F4A7C15)


def _mix(x):
    x = x ^ (x >> np.uint64(30))
    x = x * _M1
    x = x ^ (x >> np.uint64(27))
    x = x * _M2
    return x ^ (x >> np.uint64(31))


def draw(seed, step, pos, rep, attempt, m):
    """Draws in [0, m) for arrays (or scalars) of step, pos, rep and attempt; uint64 arithmetic wraps."""
    u = lambda v: np.asarray(v).astype(np.uint64)  # noqa: E731
    with np.errstate(over="ignore"):
        h = _mix(u(seed) + _G * (u(step) + np.uint64(1)))
        h = _mix(h + _G * (u(pos) + np.uint64(1)))
        h = _mix(h + _G * ((u(rep) << np.uint64(32)) + u(attempt) + np.uint64(1)))
        return (((h >> np.uint64(32)) * u(m)) >> np.uint64(32)).astype(np.int64)


def sample_negatives(indptr, cols, rows, n_items, n, *, seed, step0=0, batch_size=None, max_attempts=10, popular=False,
                     coo_items=None):
    """[len(rows), n] negatives: per (sample, rep) the first draw that is not in the user's CSR row, or the draw of
    attempt ``max_attempts``.  ``popular`` draws from ``coo_items``, the item of every interaction (default ``cols``)."""
    table = np.asarray(cols if coo_items is None else coo_items)
    rows = np.asarray(rows, dtype=np.int64)
    S = len(rows)
    batch_size = batch_size or max(S, 1)
    g = np.repeat(np.arange(S), n)
    rep = np.tile(np.arange(n), S)
    step, pos, row = step0 + g // batch_size, g % batch_size, rows[g]
    keys = np.repeat(np.arange(len(indptr) - 1, dtype=np.int64), np.diff(indptr)) * n_items + cols
    out = np.zeros(S * n, dtype=np.int32)
    todo = np.arange(S * n)
    for attempt in range(max_attempts + 1):
        d = draw(seed, step[todo], pos[todo], rep[todo], attempt, len(table) if popular else n_items)
        c = table[d] if popular else d
        out[todo] = c
        if attempt == max_attempts:
            break
        if len(keys) == 0:
            break
        k = row[todo] * n_items + c
        at = np.minimum(np.searchsorted(keys, k), len(keys) - 1)
        todo = todo[keys[at] == k]  # training interactions draw again
        if len(todo) == 0:
            break
    return out.reshape(S, n)


NAMES = ("u_bias.weight", "i_bias.weight", "u_embed.weight", "i_embed.weight")


class Model:
    """The parameter tables as leaf tensors under their state-dict names; lookups are ``F.embedding`` (with sparse
    gradients when ``sparse``, which is what ``SparseAdam`` takes)."""

    def __init__(self, params: dict, sparse: bool, dtype=torch.float32, device="cpu"):
        self.sparse = sparse
        self.tables = {
            name: torch.as_tensor(params[name]).detach().to(device, dtype).clone().requires_grad_()
            for name in NAMES
            if params.get(name) is not None
        }

    def parameters(self):
        return list(self.tables.values())

    def named_parameters(self):
        return self.tables.items()

    def state_dict(self) -> dict[str, torch.Tensor]:
        return {name: t.detach() for name, t in self.tables.items()}

    def rows(self, name: str, index: torch.Tensor) -> torch.Tensor:
        return F.embedding(index, self.tables[name], sparse=self.sparse)

    def scores_and_norms(self, users: torch.Tensor, items: torch.Tensor):
        """``users`` [B], ``items`` [B, m] -> score and regularisation norm of every (user, item), both [B, m]."""
        u = self.rows("u_embed.weight", users)  # [B, k]
        i = self.rows("i_embed.weight", items)  # [B, m, k]
        score = (u[:, None, :] * i).sum(dim=2)
        norm = u.norm(dim=1)[:, None] + i.norm(dim=2)  # plain 2-norms, not squared
        if "u_bias.weight" in self.tables:
            b = self.rows("u_bias.weight", users)[:, 0]
            score, norm = score + b[:, None], norm + (b * b)[:, None]
        if "i_bias.weight" in self.tables:
            c = self.rows("i_bias.weight", items)[:, :, 0]
            score, norm = score + c, norm + c * c
        return score, norm


def make_optimizer(model: Model, reg_method, lr: float, regularization: float):
    if reg_method == "AdamW":
        return torch.optim.AdamW(model.parameters(), lr=lr, weight_decay=regularization)
    return torch.optim.SparseAdam(model.parameters(), lr=lr)


def batch_loss(model: Model, users, pos, neg, *, loss: str, reg_method, regularization: float, positive_weight: float):
    """The batch loss of section "FlexMF implicit" of ``include/lkpy_b200.h``; -log sigmoid(x) is softplus(-x)."""
    dev = next(iter(model.tables.values())).device
    users = torch.as_tensor(users).to(dev).long().flatten()
    pos = torch.as_tensor(pos).to(dev).long().reshape(-1, 1)
    neg = torch.as_tensor(neg).to(dev).long().reshape(len(users), -1)
    s_pos, norm_pos = model.scores_and_norms(users, pos)
    s_neg, norm_neg = model.scores_and_norms(users, neg)
    if loss == "logistic":
        total = positive_weight * F.softplus(-s_pos).sum() + F.softplus(s_neg).sum()
        out = total / (s_pos.numel() + s_neg.numel())
    else:
        out = F.softplus(s_neg - s_pos).mean()  # every (positive, negative) pair of a sample
    if reg_method == "L2":
        out = out + 0.5 * regularization * (norm_pos.mean() + norm_neg.mean())
    return out


def train_step(model: Model, opt, users, pos, neg, **kw) -> float:
    out = batch_loss(model, users, pos, neg, **kw)
    out.backward()
    opt.step()
    opt.zero_grad()
    return float(out.detach())


def moments(model: Model, opt) -> dict[str, tuple[torch.Tensor, torch.Tensor]]:
    """(exp_avg, exp_avg_sq) per state-dict name, zeros before the first step."""
    out = {}
    for name, p in model.named_parameters():
        st = opt.state.get(p, {})
        out[name] = tuple(st.get(key, torch.zeros_like(p)).detach().clone() for key in ("exp_avg", "exp_avg_sq"))
    return out
