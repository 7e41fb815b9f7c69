"""
The reference's own FlexMF modules (``flexmf/_model.py``, ``_base.py``, ``_training.py``, ``_explicit.py``) on top of
the sandbox of ``ref_sandbox``, which loads ``lenskit.training``, ``lenskit.torch``, ``lenskit.config.common`` and the
data classes they import.  What the FlexMF trainers need beyond that is added here:

* ``lenskit.data.MatrixRelationshipSet`` (imported by name by ``_training.py``; not used on this path);
* ``lenskit.parallel.is_free_threaded(require_active=...)`` (``TrainingOptions.torch_compilation_enabled``);
* ``FlexMFDataset``: the slice of ``Dataset`` the trainers read besides the ALS one — the rating matrix as a torch
  COO tensor and the per-user / per-item interaction counts.
"""

from __future__ import annotations

import contextlib
import sys

import numpy as np

import ref_sandbox


class FlexMFDataset(ref_sandbox.FakeDataset):
    """``FakeDataset`` with ``interaction_matrix(format="torch", layout="coo")`` and ``user_stats`` / ``item_stats``."""

    def interaction_matrix(self, *, format: str = "scipy", layout: str = "csr", field: str | None = None, **kw):
        if format != "torch":
            return super().interaction_matrix(format=format, layout=layout, field=field, **kw)
        import torch

        assert layout == "coo"
        it = self._inter
        vals = it.ratings.astype(np.float32) if field == "rating" else np.ones(it.nnz, dtype=np.float32)
        idx = torch.from_numpy(np.stack([it.users, it.items]).astype(np.int64))
        # coalesced, in (user, item) order: the reference reads .indices() and .values()
        return torch.sparse_coo_tensor(idx, torch.from_numpy(vals), (it.n_users, it.n_items)).coalesce()

    def user_stats(self):
        import pandas as pd

        return pd.DataFrame({"count": np.bincount(self._inter.users, minlength=self._inter.n_users)})

    def item_stats(self):
        import pandas as pd

        return pd.DataFrame({"count": np.bincount(self._inter.items, minlength=self._inter.n_items)})


@contextlib.contextmanager
def flexmf_modules():
    """``ref_sandbox.reference_modules()`` plus the reference's FlexMF modules; yields ``{module name: module}``."""
    with ref_sandbox.reference_modules() as mods:
        not_free_threaded = lambda *_a, **_k: False  # noqa: E731
        sys.modules["lenskit.parallel"].is_free_threaded = not_free_threaded
        mods["lenskit.training"].is_free_threaded = not_free_threaded  # imported by name when training.py loaded
        sys.modules["lenskit.data"].MatrixRelationshipSet = type("MatrixRelationshipSet", (), {})
        ref_sandbox._module("lenskit.flexmf", package=True)
        for name, rel in (
            ("lenskit.flexmf._model", "flexmf/_model.py"),
            ("lenskit.flexmf._base", "flexmf/_base.py"),
            ("lenskit.flexmf._training", "flexmf/_training.py"),
            ("lenskit.flexmf._explicit", "flexmf/_explicit.py"),
        ):
            mods[name] = ref_sandbox._load(name, rel)
        yield mods
