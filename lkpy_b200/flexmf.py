"""
FlexMF scorers on the H100 engine — the component surface of ``lenskit.flexmf.FlexMFImplicitScorer`` and
``FlexMFExplicitScorer`` (``src/lenskit/flexmf/_implicit.py``, ``_explicit.py``, ``_base.py``, ``_training.py``,
``_model.py``): matrix factorisation trained by minibatch Adam, on the logistic or the pairwise (BPR) loss over
sampled negatives (implicit), or on the squared error of mean-centred ratings (explicit).

Same config fields, aliases, presets and defaults, the same initial parameters for a seed (torch's ``normal_`` on a
CPU generator: user bias, item bias, user embeddings, item embeddings; rows without interactions zeroed), the same
first-epoch sample order (``rng.permutation``), and the same step mathematics to rounding.  What differs:

* negatives are drawn on the device by ``lk_flexmf_sample_negatives`` from this library's counter-based generator,
  seeded once per trainer from the NumPy generator, not from the reference's PCG64 stream;
* a step is ``lk_flexmf_step`` (no autograd, no float atomics): two trainings with one seed are bit-identical;
* ``loss="warp"`` / ``negative_strategy="misranked"`` and ``convolution_layers > 0`` (LightGCN) are rejected when the
  configuration is made.

The explicit trainer draws nothing from the NumPy generator but the epoch permutations, so with the same seed its
whole sample order is the reference's.  Its model has no bias terms: the reference's ``FlexMFModel`` keeps
``u_bias = None`` / ``i_bias = None`` as class attributes, which shadow the ``nn.Embedding`` modules its constructor
registers, so ``self.u_bias is not None`` is false in ``__init__`` and ``forward``.  The bias tables it creates are
never drawn from the seeded generator, never enter a score or the L2 norm and never receive a gradient; the
embeddings take the generator's first draws.  The explicit model here computes exactly that model, ``u·i + mu``.

Inference is ``ub + ib + u·i`` (implicit) or ``u·i + mu`` (explicit): the known-user scoring and fused top-n of
:class:`factors.KnownUserScorer` (``lk_als_recommend_batch``) with the item bias as the item offset and the user bias
(or the mean) as the query offset.
"""

from __future__ import annotations

from typing import Literal

import numpy as np
import torch
from pydantic import NonNegativeInt, PositiveFloat, PositiveInt, model_validator

from . import _lib, engine
from .components import ModelTrainer, TrainingOptions, UsesTrainer, Vocabulary, _as_dataset
from .factors import EmbeddingSize, EmbeddingSizeExp, KnownUserScorer

PRESETS = {"bpr": {"loss": "pairwise", "user_bias": False, "item_bias": False}}
PARAM_NAMES = ("u_bias.weight", "i_bias.weight", "u_embed.weight", "i_embed.weight")


class FlexMFConfigBase(EmbeddingSizeExp):
    """``FlexMFConfigBase`` (``_base.py:34-95``): what the two models' configurations share."""

    embedding_size: EmbeddingSize = 64
    batch_size: PositiveInt = 8 * 1024
    learning_rate: float = 0.01
    epochs: int = 10
    regularization: float = 0.01
    reg_method: Literal["AdamW", "L2"] | None = "AdamW"


class FlexMFImplicitConfig(FlexMFConfigBase):
    preset: Literal["bpr", "warp", "lightgcn"] | None = None
    loss: Literal["logistic", "pairwise", "warp"] = "logistic"
    negative_strategy: Literal["uniform", "popular", "misranked"] | None = None
    negative_count: PositiveInt = 1
    positive_weight: PositiveFloat = 1.0
    user_bias: bool | None = None
    item_bias: bool = True
    convolution_layers: NonNegativeInt = 0

    @model_validator(mode="before")
    @classmethod
    def apply_preset(cls, data):
        if not isinstance(data, dict):
            return data
        preset = data.get("preset")
        if preset in ("warp", "lightgcn"):
            raise ValueError(f"preset={preset!r} is not covered by the engine (DESIGN.md §6)")
        if preset is not None:
            if preset not in PRESETS:
                raise ValueError(f"unknown preset '{preset}'")
            data = PRESETS[preset] | data
        return data

    @model_validator(mode="after")
    def check_covered(self):
        if self.loss == "warp":
            raise ValueError("loss='warp' is not covered by the engine (DESIGN.md §6)")
        if self.negative_strategy == "misranked":
            raise ValueError("negative_strategy='misranked' is not covered by the engine (DESIGN.md §6)")
        if self.convolution_layers > 0:
            raise ValueError("convolution_layers > 0 (LightGCN) is not covered by the engine (DESIGN.md §6)")
        return self

    def selected_negative_strategy(self) -> str:
        return self.negative_strategy or "uniform"

    def selected_user_bias(self) -> bool:
        return self.loss == "logistic" if self.user_bias is None else self.user_bias


class FlexMFExplicitConfig(FlexMFConfigBase):
    """``FlexMFExplicitConfig`` (``_explicit.py:25-35``): stronger regularisation, the L2 term by default."""

    regularization: float = 0.1
    reg_method: Literal["AdamW", "L2"] | None = "L2"


def _torch_seed(rng_input) -> int | None:
    """
    The integer a ``TrainingOptions.rng`` value seeds torch with, chosen so that the initial parameters equal the
    reference's for the same value: an integer is itself, a seed sequence (or the sequence of integers that makes
    one) gives its first 32-bit state word, a bit generator its next raw output, and a NumPy generator one draw from
    the int32 range, which moves that generator on.  ``None`` leaves torch's default seed.
    """
    if rng_input is None or isinstance(rng_input, (int, np.integer)):
        return None if rng_input is None else int(rng_input)
    if isinstance(rng_input, np.random.Generator):
        return int(rng_input.integers(-(2**31), 2**31 - 1))
    if isinstance(rng_input, np.random.BitGenerator):
        return int(rng_input.random_raw())
    words = rng_input if isinstance(rng_input, np.random.SeedSequence) else np.random.SeedSequence(rng_input)
    return int(words.generate_state(1)[0])


def _torch_generator(rng_input) -> torch.Generator:
    gen, seed = torch.Generator(), _torch_seed(rng_input)
    return gen if seed is None else gen.manual_seed(seed)


def initial_parameters(n_users: int, n_items: int, k: int, user_bias: bool, item_bias: bool, gen: torch.Generator,
                       user_counts=None, item_counts=None) -> dict[str, torch.Tensor]:  # fmt: skip
    """The reference's initial model (``_model.py:84-90``, ``_training.py:108-112``) as a state dict on the CPU."""
    shapes = {"u_bias.weight": (n_users, 1), "i_bias.weight": (n_items, 1), "u_embed.weight": (n_users, k),
              "i_embed.weight": (n_items, k)}  # fmt: skip
    have = {"u_bias.weight": user_bias, "i_bias.weight": item_bias, "u_embed.weight": True, "i_embed.weight": True}
    out = {}
    for name in PARAM_NAMES:
        if have[name]:
            out[name] = torch.nn.init.normal_(torch.empty(shapes[name], dtype=torch.float32), std=0.1, generator=gen)
    for prefix, counts in (("u_", user_counts), ("i_", item_counts)):
        if counts is not None:
            empty = torch.as_tensor(np.asarray(counts) == 0)
            for name, t in out.items():
                if name.startswith(prefix):
                    t[empty] = 0
    return out


class FlexMFScorerBase(KnownUserScorer, UsesTrainer):
    """``FlexMFScorerBase`` (``_base.py:98-164``): the known-user scoring of :class:`KnownUserScorer`
    (``__call__`` and the batched ``score_matrix`` / ``score_batch`` / ``recommend_batch``) with the biases as the
    kernel's offsets."""

    config: FlexMFConfigBase
    user_bias: np.ndarray | None = None
    item_bias: np.ndarray | None = None

    def batch_offsets(self, user_nums: np.ndarray, fold_bias):
        ub = None
        if self.user_bias is not None:
            ub = np.where(user_nums >= 0, self.user_bias[np.maximum(user_nums, 0)], 0.0).astype(np.float32)
        return self.item_bias, ub


class FlexMFImplicitScorer(FlexMFScorerBase):
    """``FlexMFImplicitScorer``: ``train`` and the scoring of :class:`FlexMFScorerBase`."""

    CONFIG_CLASS = FlexMFImplicitConfig
    config: FlexMFImplicitConfig

    def create_trainer(self, data, options):
        return FlexMFImplicitTrainer(self, data, options)


class FlexMFExplicitScorer(FlexMFScorerBase):
    """``FlexMFExplicitScorer`` (``_explicit.py:38-55``): rating prediction ``u·i + global_bias`` (the reference's
    model, whose bias terms are inactive: see the module docstring).  ``score_matrix`` / ``recommend_batch`` /
    ``score_batch`` / ``__call__`` add the item offset to the dot product, then the query offset ``ub + global_bias``;
    with the reference's model those are no item offset and ``global_bias`` rounded to f32."""

    CONFIG_CLASS = FlexMFExplicitConfig
    config: FlexMFExplicitConfig
    global_bias: float | None = None

    def create_trainer(self, data, options):
        return FlexMFExplicitTrainer(self, data, options)

    def batch_offsets(self, user_nums: np.ndarray, fold_bias):
        ib, ub = super().batch_offsets(user_nums, fold_bias)
        mu = np.float32(self.global_bias)
        return ib, (np.full(len(user_nums), mu, dtype=np.float32) if ub is None else (ub + mu).astype(np.float32))


class FlexMFTrainerBase(ModelTrainer):
    """``FlexMFTrainerBase`` (``_training.py:39-258``) with device-resident state: the data intake, the initial
    parameters, the epoch loop and the hand-back to the scorer.  Subclasses make the ``engine.FlexMFState``."""

    def __init__(self, scorer: FlexMFScorerBase, data, options: TrainingOptions):
        from .prep import DeviceInteractions

        self.scorer = scorer
        self.device = _lib.require_device()
        self.rng = options.random_generator()
        torch_rng = _torch_generator(options.rng)
        if isinstance(data, DeviceInteractions):
            scorer.users = Vocabulary(np.arange(data.n_users), "user")
            scorer.items = Vocabulary(np.arange(data.n_items), "item")
            users, items, n_users, n_items = data.users, data.items, data.n_users, data.n_items
            ratings = data.ratings
        else:
            ds = _as_dataset(data)
            scorer.users, scorer.items = ds.users, ds.items
            it = ds.interactions
            users, items, n_users, n_items = torch.from_numpy(it.users), torch.from_numpy(it.items), it.n_users, it.n_items
            ratings = None if it.ratings is None else torch.from_numpy(it.ratings)
        users, items = users.to(self.device), items.to(self.device)
        c = self.config
        params = initial_parameters(
            n_users, n_items, c.embedding_size, *self.biases(), torch_rng,
            torch.bincount(users.long(), minlength=n_users).cpu().numpy(),
            torch.bincount(items.long(), minlength=n_items).cpu().numpy(),
        )  # fmt: skip
        self.state = self.create_state(params, users, items, ratings)
        self.n_samples = int(users.numel())
        self.epochs_trained = 0  # the scorer gets its host arrays after the first epoch: until then it is not trained

    @property
    def config(self) -> FlexMFConfigBase:
        return self.scorer.config

    def biases(self) -> tuple[bool, bool]:
        """Whether the model has a user bias and an item bias."""
        raise NotImplementedError

    def create_state(self, params, users, items, ratings) -> engine.FlexMFState:
        raise NotImplementedError

    def epoch_permutation(self) -> np.ndarray:
        """The epoch's sample order, as the reference draws it (``_training.py:205-215``)."""
        return np.require(self.rng.permutation(self.n_samples), dtype=np.int32)

    def epoch_started(self) -> None:
        """Called after the epoch's permutation is drawn, before its steps."""

    def train_epoch(self) -> dict[str, float]:
        perm = self.epoch_permutation()
        self.epoch_started()
        losses = self.state.epoch(torch.from_numpy(perm))
        loss = float(losses.double().mean().item())  # the epoch's one read of the batch losses
        self.epochs_trained += 1
        self._sync_host()
        return {"loss": loss}

    def _sync_host(self) -> None:
        p = {n: t.cpu().numpy() for n, t in self.state.params.items()}
        s = self.scorer
        s.user_embeddings, s.item_embeddings = p["u_embed.weight"], p["i_embed.weight"]
        s.user_bias = p["u_bias.weight"][:, 0].copy() if "u_bias.weight" in p else None
        s.item_bias = p["i_bias.weight"][:, 0].copy() if "i_bias.weight" in p else None

    def finalize(self) -> None:
        self._sync_host()
        del self.state

    def get_parameters(self) -> dict[str, object]:
        return {n: t.cpu() for n, t in self.state.params.items()}

    def load_parameters(self, state) -> None:
        for n, t in self.state.params.items():
            t.copy_(torch.as_tensor(state[n]).to(torch.float32).reshape(t.shape))
        self._sync_host()


class FlexMFImplicitTrainer(FlexMFTrainerBase):
    """``FlexMFImplicitTrainer`` (``_implicit.py:164-290``): sampled negatives, logistic or pairwise loss."""

    config: FlexMFImplicitConfig
    _seeded = False  # the sampler seed is drawn once, in the first epoch

    def biases(self) -> tuple[bool, bool]:
        return self.config.selected_user_bias(), self.config.item_bias

    def create_state(self, params, users, items, ratings) -> engine.FlexMFState:
        c = self.config
        return engine.FlexMFState(
            params, users, items, loss=c.loss, reg_method=c.reg_method, negative_count=c.negative_count,
            popular=c.selected_negative_strategy() == "popular", batch_size=c.batch_size,
            learning_rate=c.learning_rate, regularization=c.regularization, positive_weight=c.positive_weight,
            device=self.device,
        )  # fmt: skip

    def epoch_started(self) -> None:
        if not self._seeded:
            # after the first permutation, so that the first epoch's order is the reference's for the same seed
            self.state.seed = int(self.rng.integers(0, 2**63))
            self._seeded = True


class FlexMFExplicitTrainer(FlexMFTrainerBase):
    """``FlexMFExplicitTrainer`` (``_explicit.py:58-125``): squared error on the ratings less their mean, no
    negatives, and no bias terms, as in the reference's model."""

    config: FlexMFExplicitConfig

    def biases(self) -> tuple[bool, bool]:
        return False, False

    def create_state(self, params, users, items, ratings) -> engine.FlexMFState:
        if ratings is None:
            raise ValueError("FlexMFExplicitScorer trains on ratings, and the data has none")
        # the reference's f32 torch mean on the host (_explicit.py:72-79), and the targets r - mu
        values = ratings.cpu().to(torch.float32)
        mean = values.mean()
        self.scorer.global_bias = mean.item()
        c = self.config
        return engine.FlexMFState(
            params, users, items, loss="mse", reg_method=c.reg_method, negative_count=0, batch_size=c.batch_size,
            learning_rate=c.learning_rate, regularization=c.regularization, ratings=values - mean, device=self.device,
        )  # fmt: skip
