"""
Plain restatement of the FlexMF explicit training pieces, for the tests, ``smoke()`` and ``tools/flexmf_bench.py``,
on top of the implicit model's restatement (``flexmf_oracle``: the parameter tables, the optimisers):

* ``mse_terms`` / ``batch_loss`` / ``train_step``: one minibatch step of the explicit model in plain torch — embedding
  lookups, the squared error of the centred ratings, the L2 term, ``backward()`` and ``torch.optim.AdamW`` /
  ``SparseAdam`` — parameterised on dtype;
* ``explicit_epoch``: the explicit trainer's epoch (``_training.py:157-215``) over those steps.
"""

from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

import flexmf_oracle as fo


def mse_terms(model: fo.Model, users, items, ratings, *, reg_method, regularization: float):
    """The explicit model's step (``_explicit.py:108-125``): (what is differentiated, the squared error alone, which
    is the batch loss reported).  With L2 the differentiated loss adds ``regularization * mean_b(norm_b)``."""
    dev = next(iter(model.tables.values())).device
    users = torch.as_tensor(users).to(dev).long().flatten()
    items = torch.as_tensor(items).to(dev).long().reshape(-1, 1)
    score, norm = model.scores_and_norms(users, items)
    t = torch.as_tensor(ratings).to(dev, score.dtype).flatten()
    err = F.mse_loss(score[:, 0], t)
    if reg_method == "L2":
        return err + norm[:, 0].mean() * regularization, err
    return err, err


def batch_loss(model: fo.Model, users, items, ratings, *, reg_method, regularization: float):
    """The batch loss of the MSE branch of section "FlexMF" of ``include/lkpy_b200.h``: the squared error alone,
    without the norm term."""
    return mse_terms(model, users, items, ratings, reg_method=reg_method, regularization=regularization)[1]


def train_step(model: fo.Model, opt, users, items, ratings, *, reg_method, regularization: float) -> float:
    """One step; the batch loss (the squared error alone, as the reference reports it)."""
    out, reported = mse_terms(model, users, items, ratings, reg_method=reg_method, regularization=regularization)
    out.backward()
    opt.step()
    opt.zero_grad()
    return float(reported.detach())


def explicit_epoch(model: fo.Model, opt, users, items, targets, perm, batch_size: int, *, reg_method,
                   regularization: float) -> list[float]:  # fmt: skip
    """One epoch of the explicit trainer: the samples in the order ``perm``, cut into batches of ``batch_size``;
    the batch losses."""
    users, items, targets = (np.asarray(x)[perm] for x in (users, items, targets))
    out = []
    for lo in range(0, len(perm), batch_size):
        sl = slice(lo, lo + batch_size)
        out.append(train_step(model, opt, users[sl], items[sl], torch.from_numpy(targets[sl]), reg_method=reg_method,
                              regularization=regularization))  # fmt: skip
    return out
