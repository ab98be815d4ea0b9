"""``B200Recommender``: the drop-in for ``BotorchRecommender`` on purely discrete search spaces.

Mirrors the reference's call chain
  BayesianRecommender.recommend            /root/reference/baybe/recommenders/pure/bayesian/base.py:129-197
  PureRecommender._recommend_with_discrete_parts          recommenders/pure/base.py:248-307
  recommend_discrete_without_subsets       recommenders/pure/bayesian/botorch/discrete.py:78-142
with ``botorch.optim.optimize_acqf_discrete`` (sequential greedy, ``unique=True``, first maximum
wins) replaced by the CUDA engine: round 1 is one fused pass (posterior + acquisition + arg-max),
later rounds score [candidate; pending] jointly.  The candidate matrix is cached on the device per
discrete subspace (SURVEY.md row f3) and recommendations come back as row *positions*, so neither
the per-call re-encoding (discrete.py:123) nor the float-equality merge (discrete.py:133-140) of
the reference is needed.

Multi-GPU: when ``torch.distributed`` is initialised (one process per GPU), every rank scores a
contiguous row shard and the packed (score, lowest index) keys are max-reduced per greedy round by
``bb_allreduce_best`` over NVLink peer memory (``baybe_b200/peers.py``; SURVEY.md 8e).  A rank only ever holds
its own shard; the features of a round's winner are broadcast from the rank that owns it.
"""

from __future__ import annotations

import weakref
from typing import ClassVar

import numpy as np
import pandas as pd
import torch
from attrs import define, field
from attrs.converters import optional

from baybe_b200.acquisition import (AcquisitionFunction, IncompatibleAcquisitionFunctionError,
                                    convert_acqf, qLogExpectedImprovement)
from baybe_b200._lib import NEI_KINDS
from baybe_b200.bits import pack_bits
from baybe_b200.engine import DEFAULT_MC_SAMPLES, AcqConfig, DeviceGP, sobol_normal_samples, unpack_best
from baybe_b200.surrogates import GaussianProcessSurrogate

__all__ = ["B200Recommender", "NotEnoughPointsLeftError", "shard_bounds", "greedy_select",
           "recommend_discrete_positions"]


class NotEnoughPointsLeftError(Exception):
    """Same name/meaning as baybe.exceptions.NotEnoughPointsLeftError (pure/base.py:294-298)."""


def _draw_sampler_seed() -> int:
    """botorch's MC samplers draw their seed from torch's global RNG at construction
    (SURVEY.md A.6), which is how ``Settings(random_seed=...)`` makes recommendations
    reproducible (baybe/utils/random.py:124-130)."""
    return int(torch.randint(0, 1_000_000, (1,)).item())


def shard_bounds(n_rows: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous row block [lo, hi) of shard `rank` out of `world` (ceil-sized blocks)."""
    per = -(-n_rows // world)
    lo = min(rank * per, n_rows)
    return lo, min(lo + per, n_rows)


def _dist_info() -> tuple[int, int]:
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def _broadcast_seed(seed: int, device) -> int:
    """Every rank must score its shard with the SAME base samples, or the all-reduced arg-max compares values
    that are not comparable (ranks are usually seeded seed+rank): rank 0's draw wins."""
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        t = torch.tensor([seed], dtype=torch.int64,
                         device=device if dist.get_backend() == "nccl" else torch.device("cpu"))
        dist.broadcast(t, src=0)
        seed = int(t.item())
    return seed


def _allreduce_key(key: torch.Tensor) -> torch.Tensor:
    """Global maximum of the ranks' packed (score, lowest index) keys.  Device keys go through
    ``bb_allreduce_best`` (baybe_b200/peers.py: one warp per rank, NVLink peer atomics, enqueued on the stream --
    no host-issued collective); host keys (the gloo protocol tests) through ``dist.all_reduce``."""
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        if key.is_cuda:
            from baybe_b200.peers import get_peer_reduce

            return get_peer_reduce(key.device).allreduce_best(key)
        dist.all_reduce(key, op=dist.ReduceOp.MAX)
    return key


def merge_topk_across_ranks(vals: torch.Tensor, idx: torch.Tensor, k: int) -> tuple[torch.Tensor, torch.Tensor]:
    """Global top-k from every rank's local top-k (SURVEY.md 8e, BASELINE config 5 "NCCL top-k argmax"): one
    all-gather of k (value, global index) pairs per rank, then a k-way merge on every rank.  Ties go to the lowest
    global index, like ``bb_topk`` / ``torch.argmax``.  `vals`/`idx`: this rank's best k (fewer entries may be
    padded with -inf / -1); the tensors stay on their device (NCCL for CUDA tensors, gloo on the CPU)."""
    import torch.distributed as dist

    vals = vals.reshape(-1).to(torch.float32)
    idx = idx.reshape(-1).to(torch.int64)
    if vals.numel() != k or idx.numel() != k:
        raise ValueError(f"expected {k} local candidates, got {vals.numel()} values / {idx.numel()} indices")
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        world = dist.get_world_size()
        all_v = [torch.empty_like(vals) for _ in range(world)]
        all_i = [torch.empty_like(idx) for _ in range(world)]
        dist.all_gather(all_v, vals)
        dist.all_gather(all_i, idx)
        vals, idx = torch.cat(all_v), torch.cat(all_i)
    valid = idx >= 0
    v = torch.where(valid, vals, torch.full_like(vals, -float("inf")))
    # order by (value desc, index asc): stable sort by index first, then by value
    order = torch.argsort(torch.where(valid, idx, torch.full_like(idx, torch.iinfo(torch.int64).max)), stable=True)
    order = order[torch.argsort(v[order], descending=True, stable=True)]
    top = order[:k]
    return v[top], torch.where(valid[top], idx[top], torch.full_like(idx[top], -1))


def distributed_topk(scores: torch.Tensor, keep: torch.Tensor | None, k: int, offset: int = 0):
    """Top-k of a row-sharded score vector: per-rank ``bb_topk`` on the device, then ``merge_topk_across_ranks``."""
    v, i = torch.ops.baybe_b200.topk(scores, keep, k)
    i = torch.where(i >= 0, i + int(offset), i)
    return merge_topk_across_ranks(v, i, k)


def _scores_for(gp: DeviceGP, cfg: AcqConfig, x: torch.Tensor, pending: np.ndarray | None, seed: int,
                n_samples: int) -> torch.Tensor:
    """Per-candidate acquisition values (q=1 batches, optionally joint with pending points)."""
    if pending is not None and len(pending) > 0:
        z = sobol_normal_samples(n_samples, 1 + len(pending), seed)
        return gp.score_joint(cfg, x, pending, z)
    z = sobol_normal_samples(n_samples, 1, seed)[:, 0] if cfg.is_mc else None
    scores, _ = gp.score(cfg, x, z)
    return scores


def _winner_row(x_shard: torch.Tensor, d: int, idx: int, offset: int) -> np.ndarray:
    """Comp-rep row (float64, length d) of the global position `idx`: read from the device shard of the rank
    that owns it and broadcast to the others (d floats) -- no rank needs the whole matrix on its host
    (at BASELINE config 4 that would be 10M x 2048 x 8 B = 164 GB per rank)."""
    import torch.distributed as dist

    from baybe_b200.bits import unpack_bits

    rank, world = _dist_info()
    mine = offset <= idx < offset + x_shard.shape[0]
    row = torch.zeros(d, dtype=torch.float64, device=x_shard.device)
    if mine:
        r = x_shard[idx - offset]
        if x_shard.dtype == torch.uint8:
            row = torch.from_numpy(unpack_bits(r.reshape(1, -1).cpu().numpy(), d)[0]).to(x_shard.device, torch.float64)
        else:
            row = r.to(torch.float64)
    if world > 1:
        owner = torch.tensor([rank if mine else -1], dtype=torch.int64, device=x_shard.device)
        dist.all_reduce(owner, op=dist.ReduceOp.MAX)
        dist.broadcast(row, src=int(owner.item()))
    return row.cpu().numpy()


def greedy_select(gp: DeviceGP, cfg: AcqConfig, x_shard: torch.Tensor, d: int, q: int,
                  base_pending: np.ndarray | None, seed: int, n_samples: int = DEFAULT_MC_SAMPLES,
                  offset: int = 0, keep_init: torch.Tensor | None = None) -> tuple[list[int], list[float]]:
    """Sequential greedy selection of q rows (global positions) -- ``optimize_acqf_discrete`` with
    ``unique=True``.  `x_shard` holds this rank's rows [offset, offset+len) on the device; the features of each
    round's winner are fetched from the rank that owns it (``_winner_row``).  A `gp` with a ``round_best`` method
    (``baybe_b200.multiobjective.HviScorer``, ``baybe_b200.objectives.ObjectiveScorer``, ``baybe_b200.noisy.NeiScorer``)
    scores a round itself and maps the winner's key value to the reported acquisition value."""
    chosen: list[int] = []
    values: list[float] = []
    keep = (torch.ones(x_shard.shape[0], dtype=torch.uint8, device=x_shard.device)
            if keep_init is None else keep_init.to(device=x_shard.device, dtype=torch.uint8).clone())
    pend = np.zeros((0, d)) if base_pending is None else np.asarray(base_pending, dtype=np.float64).reshape(-1, d)
    round_best = getattr(gp, "round_best", None)
    for r in range(q):
        report = None
        if round_best is not None:
            key, report = round_best(x_shard, pend, keep, offset, seed, n_samples)
        elif len(pend) == 0:
            z = sobol_normal_samples(n_samples, 1, seed)[:, 0] if cfg.is_mc else None
            _, key = gp.score(cfg, x_shard, z, keep=keep, index_offset=offset, want_scores=False)
        else:
            z = sobol_normal_samples(n_samples, 1 + len(pend), seed)
            scores = gp.score_joint(cfg, x_shard, pend, z)
            key = gp.argmax(scores, keep, offset)
        key = _allreduce_key(key)
        val, idx = unpack_best(int(key.item()))
        if idx < 0:
            raise NotEnoughPointsLeftError("no eligible candidate left to recommend")
        chosen.append(idx)
        values.append(val if report is None else report(val))
        if offset <= idx < offset + x_shard.shape[0]:
            keep[idx - offset] = 0
        if r + 1 < q:
            pend = np.concatenate([pend, _winner_row(x_shard, d, idx, offset).reshape(1, d)], axis=0)
    return chosen, values


# comp-reps that are all 0/1 and at least this wide (always a wide-feature model: n_pad*d*4 > 56 KB) are kept
# bit-packed on the device
BITS_MIN_COLUMNS = 256


class _DeviceCache:
    """comp-rep matrices resident on the GPU, keyed by the identity of the subspace's cached
    ``comp_rep`` dataframe (attrs classes with ``eq=True`` are unhashable, dataframes are
    weak-referenceable); an entry dies with its dataframe."""

    def __init__(self):
        self._store: dict[int, tuple] = {}

    def get(self, subspace, device, lo: int, hi: int) -> tuple[torch.Tensor, int]:
        """(device shard rows [lo, hi), number of comp-rep columns).  Only the shard is converted: a rank never
        materialises rows it does not own (VERDICT r1, weak #10)."""
        comp_df = subspace.comp_rep
        key = id(comp_df)
        entry = self._store.get(key)
        if entry is None or entry[0]() is not comp_df or entry[1] != (str(device), lo, hi):
            shard = np.ascontiguousarray(comp_df.iloc[lo:hi].to_numpy(dtype=np.float64))
            if shard.shape[1] >= BITS_MIN_COLUMNS and bool(((shard == 0.0) | (shard == 1.0)).all()):
                # binary fingerprint space: 1 bit per feature on the device (BB_BITS_U8), 32x less HBM
                dev = torch.from_numpy(pack_bits(shard)).to(device=device)
            else:
                dev = torch.from_numpy(shard).to(device=device, dtype=torch.float32)
            ref = weakref.ref(comp_df, lambda _r, k=key: self._store.pop(k, None))
            entry = (ref, (str(device), lo, hi), dev, int(comp_df.shape[1]))
            self._store[key] = entry
        return entry[2], entry[3]


_cache = _DeviceCache()


def recommend_discrete_positions(gp: DeviceGP, cfg: AcqConfig, subspace_discrete, candidates_exp: pd.DataFrame,
                                 batch_size: int, searchspace, pending_experiments, n_mc_samples: int,
                                 acq_values_out: list | None = None) -> pd.Index:
    """``recommend_discrete_without_subsets`` (botorch/discrete.py:78-142) on the engine: candidate rows are the
    device-resident comp-rep shard of the subspace, a filtered candidate set (``FilteredSubspaceDiscrete``,
    ``Campaign.recommend`` campaign.py:549-572) becomes a position mask, and the winners come back as index
    labels of ``candidates_exp`` -- no re-encoding (discrete.py:123) and no float merge (discrete.py:133-140)."""
    rank, world = _dist_info()
    n_rows = len(subspace_discrete.comp_rep)
    lo, hi = shard_bounds(n_rows, rank, world)
    x_dev, d = _cache.get(subspace_discrete, gp.device, lo, hi)
    keep_init = None
    comp_index = subspace_discrete.comp_rep.index
    if len(candidates_exp) != n_rows or not candidates_exp.index.equals(comp_index):
        # a filtered candidate set: mask rows by position
        pos = comp_index.get_indexer(candidates_exp.index)
        if (pos < 0).any():
            raise ValueError("candidates_exp contains rows that are not part of the discrete subspace")
        mask = np.zeros(n_rows, dtype=np.uint8)
        mask[pos] = 1
        keep_init = torch.from_numpy(mask[lo:hi])
    pend = None
    if pending_experiments is not None and len(pending_experiments) > 0:
        pend = searchspace.transform(pending_experiments, allow_extra=True).to_numpy(dtype=np.float64)
    seed = _broadcast_seed(_draw_sampler_seed(), gp.device)
    positions, vals = greedy_select(gp, cfg, x_dev, d, batch_size, pend, seed, n_mc_samples, offset=lo,
                                    keep_init=keep_init)
    if acq_values_out is not None:
        acq_values_out[:] = vals
    return comp_index[np.asarray(positions, dtype=np.int64)]


@define
class B200Recommender:
    """Bayesian recommender for discrete search spaces running on the B200 engine."""

    compatibility: ClassVar[str] = "DISCRETE"
    supports_discrete_subset_generating_constraints: ClassVar[bool] = False

    surrogate_model: GaussianProcessSurrogate = field(factory=GaussianProcessSurrogate)
    acquisition_function: AcquisitionFunction | None = field(default=None, converter=optional(convert_acqf))
    n_mc_samples: int = field(default=DEFAULT_MC_SAMPLES)

    _objective = field(init=False, default=None, eq=False, repr=False)
    _context = field(init=False, default=None, eq=False, repr=False)
    _scorer = field(init=False, default=None, eq=False, repr=False)
    _last_acq_values: list = field(init=False, factory=list, eq=False, repr=False)

    def _get_acquisition_function(self, objective) -> AcquisitionFunction:
        """Default acquisition function: qLogEI (bayesian/base.py:70-74)."""
        return qLogExpectedImprovement() if self.acquisition_function is None else self.acquisition_function

    def get_surrogate(self, searchspace, objective, measurements) -> GaussianProcessSurrogate:
        self.surrogate_model.fit(searchspace, objective, measurements)
        return self.surrogate_model

    def recommend(self, batch_size: int, searchspace, objective=None, measurements: pd.DataFrame | None = None,
                  pending_experiments: pd.DataFrame | None = None) -> pd.DataFrame:
        """Rows of ``searchspace.discrete.exp_rep`` with their original index
        (RecommenderProtocol, recommenders/base.py:11-48)."""
        if objective is None:
            raise NotImplementedError(
                f"Recommenders of type '{type(self).__name__}' require that an objective is specified.")
        if measurements is None or measurements.empty:
            raise NotImplementedError(
                f"Recommenders of type '{type(self).__name__}' do not support empty training data.")
        acqf = self._get_acquisition_function(objective)
        if batch_size > 1 and not acqf.supports_batching:
            raise IncompatibleAcquisitionFunctionError(
                f"The '{type(self).__name__}' only works with Monte Carlo acquisition functions "
                f"for batch sizes > 1.")
        from baybe_b200.objectives import uses_objective_scorer

        self._objective = objective
        surrogate = self.get_surrogate(searchspace, objective, measurements)
        self._scorer = None
        # a single target with a non-affine transformation, or the noisy-EI family
        if uses_objective_scorer(objective) or acqf.abbreviation in NEI_KINDS:
            if pending_experiments is not None and not acqf.supports_pending_experiments:
                raise IncompatibleAcquisitionFunctionError(
                    f"The chosen acquisition function of type '{type(acqf).__name__}' "
                    f"does not support pending experiments.")
            self._scorer = acqf.scorer(surrogate, searchspace, objective, measurements)
            cfg = self._scorer.cfg
        else:
            cfg = acqf.to_engine(surrogate, searchspace, objective, measurements, pending_experiments)
        subspace = searchspace.discrete
        candidates_exp, _ = subspace.get_candidates()
        if len(candidates_exp) < batch_size:
            raise NotEnoughPointsLeftError(
                f"Using the current settings, there are fewer than {batch_size} possible data points "
                f"left to recommend.")
        self._context = (cfg, searchspace, pending_experiments)
        idxs = self._recommend_discrete(subspace, candidates_exp, batch_size)
        return subspace.exp_rep.loc[idxs, :]

    def _recommend_discrete(self, subspace_discrete, candidates_exp: pd.DataFrame, batch_size: int) -> pd.Index:
        """Same hook signature as ``PureRecommender._recommend_discrete`` (pure/base.py:142-180,
        botorch/core.py:156-184); the recommendation context (acquisition config, search space, pending
        experiments) was stored by ``recommend`` the way the reference stores ``_botorch_acqf``."""
        cfg, searchspace, pending_experiments = self._context
        gp = self._scorer if self._scorer is not None else self.surrogate_model.device_gp
        return recommend_discrete_positions(gp, cfg, subspace_discrete, candidates_exp,
                                            batch_size, searchspace, pending_experiments, self.n_mc_samples,
                                            self._last_acq_values)

    def acquisition_values(self, candidates: pd.DataFrame, searchspace, objective, measurements,
                           pending_experiments: pd.DataFrame | None = None,
                           acquisition_function: AcquisitionFunction | None = None) -> pd.Series:
        """Acquisition value of every candidate (bayesian/base.py:199-237)."""
        surrogate = self.get_surrogate(searchspace, objective, measurements)
        acqf = acquisition_function or self._get_acquisition_function(objective)
        return acqf.evaluate(candidates, surrogate, searchspace, objective, measurements,
                             pending_experiments, jointly=False)

    def joint_acquisition_value(self, candidates: pd.DataFrame, searchspace, objective, measurements,
                                pending_experiments: pd.DataFrame | None = None,
                                acquisition_function: AcquisitionFunction | None = None) -> float:
        """Joint acquisition value of the whole candidate batch (bayesian/base.py:239-277)."""
        surrogate = self.get_surrogate(searchspace, objective, measurements)
        acqf = acquisition_function or self._get_acquisition_function(objective)
        return acqf.evaluate(candidates, surrogate, searchspace, objective, measurements,
                             pending_experiments, jointly=True)
