"""Drop-in binding for the real ``baybe`` package: a ``BayesianRecommender`` subclass that BayBE's own
``Campaign`` drives unchanged, with the recommend-time hot path on the B200 engine.

Importing this module needs ``baybe`` (it subclasses BayBE's classes); nothing else in ``baybe_b200`` does.

What it satisfies (paths under ``/root/reference/baybe``):
  * ``isinstance(recommender, BayesianRecommender)`` -- the gate ``Campaign.get_surrogate`` / ``posterior_stats`` /
    ``acquisition_values`` / ``joint_acquisition_value`` check (``campaign.py:750-754,798-807,864-899``);
  * the ``PureRecommender`` hook ``_recommend_discrete(subspace_discrete, candidates_exp, batch_size) -> pd.Index``
    with the reference's exact signature (``recommenders/pure/base.py:142-180``, ``botorch/core.py:156-184``);
  * ``compatibility`` / ``supports_discrete_subset_generating_constraints`` class flags
    (``recommenders/pure/base.py:34-60``), subset-generating constraints handled like
    ``recommend_discrete_with_subsets`` (``botorch/discrete.py:21-75``): greedy selection inside every subset, the
    batch with the highest JOINT acquisition value wins;
  * ``FilteredSubspaceDiscrete`` candidate sets produced by ``Campaign.recommend`` from its metadata masks
    (``campaign.py:549-572``, ``searchspace/_filtered.py:41-43``) become position masks on the device-resident
    comp-rep matrix -- no re-encoding, no float merge;
  * ``get_acquisition_function`` returns a callable with the contract BayBE relies on (``X[b, q, d] -> [b]``,
    ``X_pending`` / ``set_X_pending``, ``model``; ``botorch/discrete.py:68,125``), evaluated by the engine.

The surrogate is ``baybe_b200.GaussianProcessSurrogate`` (``SurrogateProtocol``: ``fit`` + ``posterior`` /
``posterior_stats``); BayBE's acquisition-function *specs* (``baybe.acquisition.qLogEI`` ...) are accepted as they are
and mapped onto the engine's kinds by their ``abbreviation``.
"""
from __future__ import annotations

from typing import ClassVar

import numpy as np
import pandas as pd
import torch
from attrs import define, field, fields_dict
from attrs.validators import ge, instance_of

from baybe.exceptions import (IncompatibilityError, IncompatibleAcquisitionFunctionError,  # noqa: E402
                              InfeasibilityError)
from baybe.recommenders.pure.bayesian.base import BayesianRecommender
from baybe.searchspace import SearchSpaceType

from baybe_b200 import _lib
from baybe_b200 import acquisition as _acq
from baybe_b200.engine import DEFAULT_MC_SAMPLES, sobol_normal_samples
from baybe_b200.recommenders import _draw_sampler_seed, recommend_discrete_positions
from baybe_b200.surrogates import GaussianProcessSurrogate

__all__ = ["B200BotorchRecommender", "EngineAcquisitionFunction", "mirror_acquisition_function"]


def mirror_acquisition_function(acqf) -> _acq.AcquisitionFunction:
    """BayBE acquisition spec (``baybe/acquisition/acqfs.py``) -> the engine-side spec of the same abbreviation,
    carrying over the fields both define (``beta``, ``maximize``)."""
    if isinstance(acqf, _acq.AcquisitionFunction):
        return acqf
    if isinstance(acqf, str):
        return _acq.convert_acqf(acqf)
    abbr = getattr(type(acqf), "abbreviation", None)
    if abbr is None or abbr not in _acq._BY_NAME:
        raise IncompatibleAcquisitionFunctionError(
            f"The acquisition function '{type(acqf).__name__}' is not implemented by the B200 engine "
            f"(available: {sorted({c.abbreviation for c in _acq._BY_NAME.values()})}).")
    cls = _acq._BY_NAME[abbr]
    kwargs = {k: getattr(acqf, k) for k in fields_dict(cls) if hasattr(acqf, k)}
    return cls(**kwargs)


def _integration_points(acqf, spec, searchspace) -> dict:
    """qNIPV given as BayBE's spec: its own draw of the integration points, so that Random and FPS pick exactly the
    rows BayBE picks (keyword arguments for the engine spec's ``scorer`` / ``evaluate``; empty otherwise)."""
    if spec.abbreviation in _lib.NIPV_KINDS and hasattr(acqf, "get_integration_points"):
        return {"integration": acqf.get_integration_points(searchspace)}
    return {}


class EngineAcquisitionFunction:
    """The acquisition callable BayBE hands around (``recommender._botorch_acqf``): ``acqf(X)`` with ``X`` of shape
    ``[b, q, d]`` (un-scaled comp-rep) returns ``[b]`` joint values of ``[X_b ; X_pending]``."""

    def __init__(self, surrogate: GaussianProcessSurrogate, cfg, n_mc_samples: int, X_pending=None, scorer=None):
        self.model = surrogate
        self.cfg = cfg
        self.n_mc_samples = n_mc_samples
        self.X_pending = X_pending
        # what the fused path does not serve: baybe_b200.multiobjective.HviScorer (Pareto),
        # baybe_b200.objectives.ObjectiveScorer (desirability, non-affine single targets) or
        # baybe_b200.noisy.NeiScorer (qNEI / qLogNEI on discrete spaces), baybe_b200.parego.ParegoScorer (qLogNParEGO)
        # or baybe_b200.nehvi.NehviScorer (qNEHVI)
        self.scorer = scorer
        self.seed = _draw_sampler_seed()  # botorch samplers draw their seed once, at construction

    def set_X_pending(self, X_pending=None) -> None:
        self.X_pending = X_pending

    def __call__(self, X: torch.Tensor) -> torch.Tensor:
        if X.dim() == 2:
            X = X.unsqueeze(0)
        b, q, d = X.shape
        pend = None if self.X_pending is None else torch.as_tensor(self.X_pending).reshape(-1, d)
        if self.scorer is not None:
            if q == 1 and (pend is None or len(pend) == 0):
                return torch.from_numpy(self.scorer.scores(X[:, 0, :], None, self.seed, self.n_mc_samples))
            if not self.scorer.cfg.is_mc:
                raise IncompatibleAcquisitionFunctionError("analytic acquisition functions value single points only")
            out = torch.empty(b, dtype=torch.float64)
            pn = None if pend is None or len(pend) == 0 else pend.cpu().numpy()
            for i in range(b):
                out[i] = self.scorer.joint_value(X[i].cpu().numpy(), pn, self.seed, self.n_mc_samples)
            return out
        gp = self.model.device_gp
        if q == 1 and (pend is None or len(pend) == 0):
            z = sobol_normal_samples(self.n_mc_samples, 1, self.seed)[:, 0] if self.cfg.is_mc else None
            scores, _ = gp.score(self.cfg, X[:, 0, :], z)
            return scores.to(torch.float64)
        if not self.cfg.is_mc:
            raise IncompatibleAcquisitionFunctionError("analytic acquisition functions value single points only")
        out = torch.empty(b, dtype=torch.float64)
        for i in range(b):  # candidate first, then the rest of the batch and the pending points
            rest = X[i, 1:, :] if pend is None else torch.cat([X[i, 1:, :], pend.to(X)], dim=0)
            z = sobol_normal_samples(self.n_mc_samples, 1 + len(rest), self.seed)
            out[i] = float(gp.score_joint(self.cfg, X[i, :1, :], rest.cpu().numpy(), z)[0])
        return out


@define(kw_only=True)
class B200BotorchRecommender(BayesianRecommender):
    """``BotorchRecommender`` for discrete search spaces with the scoring path on the B200 engine."""

    compatibility: ClassVar[SearchSpaceType] = SearchSpaceType.HYBRID
    supports_discrete_subset_generating_constraints: ClassVar[bool] = True

    _surrogate_model = field(alias="surrogate_model", factory=GaussianProcessSurrogate)
    """The surrogate: ``baybe_b200.GaussianProcessSurrogate`` (duck-typed ``SurrogateProtocol``)."""

    n_mc_samples: int = field(default=DEFAULT_MC_SAMPLES, validator=instance_of(int))
    """Base samples of the Monte Carlo acquisition functions (botorch's default sample shape)."""

    max_n_subsets: int = field(default=10, validator=[instance_of(int), ge(1)])
    """As ``BotorchRecommender.max_n_subsets`` (botorch/core.py:101-105)."""

    _context = field(default=None, init=False, eq=False, repr=False)
    _scorer = field(default=None, init=False, eq=False, repr=False)
    """Objectives the fused path does not serve: the ``HviScorer`` (Pareto) or ``ObjectiveScorer`` (desirability,
    non-affine single targets) set up by ``_setup_botorch_acqf``; on discrete spaces also the ``NeiScorer`` of qNEI /
    qLogNEI (its ``n_dropped``: baseline winners left out by the last evaluation)."""
    _last_acq_values: list = field(factory=list, init=False, eq=False, repr=False)

    # ---- multi-target objectives (SURVEY.md 8f-4, surrogates/composite.py:59-181) ------------------------------
    def get_surrogate(self, searchspace, objective, measurements):
        """The reference replicates single-output ``Surrogate`` subclasses per modelled quantity
        (``bayesian/base.py:35-39``); the engine surrogate is a duck-typed ``SurrogateProtocol``, so the same
        replication is done here -- with BayBE's OWN ``CompositeSurrogate``, which only needs ``fit`` and
        ``posterior_stats`` of its members.  This happens whenever the objective models more than one quantity
        (``Objective._is_multi_model``: Pareto objectives and desirability objectives that are not applied as a
        pre-transformation).  Pareto objectives recommend with qEHVI / qLogEHVI (``baybe_b200.multiobjective``),
        qNEHVI (``baybe_b200.nehvi``) or qLogNParEGO (``baybe_b200.parego``), desirability objectives with
        ``baybe_b200.objectives``."""
        multi_model = getattr(objective, "_is_multi_model", objective.is_multi_output)
        if multi_model and isinstance(self._surrogate_model, GaussianProcessSurrogate):
            from baybe.surrogates.composite import CompositeSurrogate

            self._surrogate_model = CompositeSurrogate.from_replication(self._surrogate_model)
        return super().get_surrogate(searchspace, objective, measurements)

    # ---- acquisition set-up: the engine config takes the place of the botorch acquisition function ----------
    def _setup_botorch_acqf(self, searchspace, objective, measurements, pending_experiments=None) -> None:
        self._objective = objective
        acqf = self._get_acquisition_function(objective)
        self._scorer = None
        if objective.is_multi_output:
            if getattr(type(acqf), "abbreviation", None) not in _lib.HVI_KINDS + _lib.PAREGO_KINDS + _lib.NEHVI_KINDS:
                raise IncompatibleAcquisitionFunctionError(
                    f"recommending for multi-output objectives on the B200 engine needs "
                    f"qExpectedHypervolumeImprovement (qEHVI), qLogExpectedHypervolumeImprovement (qLogEHVI), "
                    f"qNoisyExpectedHypervolumeImprovement (qNEHVI) or qLogNParEGO; "
                    f"'{type(acqf).__name__}' is not implemented (the default for multi-output objectives is "
                    f"qLogNEHVI, bayesian/base.py:73)")
        surrogate = self.get_surrogate(searchspace, objective, measurements)
        spec = mirror_acquisition_function(acqf)
        if spec.uses_scorer(objective, searchspace):
            if pending_experiments is not None and not spec.supports_pending_experiments:
                raise IncompatibleAcquisitionFunctionError(
                    f"The chosen acquisition function of type '{type(spec).__name__}' "
                    f"does not support pending experiments.")
            self._scorer = spec.scorer(surrogate, searchspace, objective, measurements,
                                       **_integration_points(acqf, spec, searchspace))
            cfg = self._scorer.cfg
        else:
            cfg = spec.to_engine(surrogate, searchspace, objective, measurements, pending_experiments)
        self._context = (cfg, searchspace, pending_experiments)
        pend = None
        if pending_experiments is not None and len(pending_experiments) > 0:
            pend = torch.from_numpy(searchspace.transform(pending_experiments, allow_extra=True)
                                    .to_numpy(dtype=np.float64))
        self._botorch_acqf = EngineAcquisitionFunction(surrogate, cfg, self.n_mc_samples, pend, scorer=self._scorer)

    # ---- the PureRecommender hook (exact reference signature) ------------------------------------------------
    def _recommend_discrete(self, subspace_discrete, candidates_exp: pd.DataFrame, batch_size: int) -> pd.Index:
        assert self._objective is not None and self._context is not None
        acqf = self._get_acquisition_function(self._objective)
        if batch_size > 1 and not acqf.supports_batching:
            raise IncompatibleAcquisitionFunctionError(
                f"The '{self.__class__.__name__}' only works with Monte Carlo "
                f"acquisition functions for batch sizes > 1.")
        if batch_size > 1 and type(acqf).__name__ == "qThompsonSampling":
            raise IncompatibilityError("Thompson sampling currently only supports a batch size of 1.")
        if subspace_discrete.n_subsets > 0:
            return self._recommend_discrete_with_subsets(subspace_discrete, candidates_exp, batch_size)
        return self._recommend_discrete_without_subsets(subspace_discrete, candidates_exp, batch_size)

    # ---- hybrid spaces (botorch/core.py:221-250 -> hybrid.py:30-161): search by scoring on the device -----------
    def _recommend_hybrid(self, searchspace, candidates_exp: pd.DataFrame, batch_size: int) -> pd.DataFrame:
        from baybe_b200.hybrid import recommend_hybrid

        assert self._objective is not None and self._context is not None
        cfg, _, pending = self._context
        if cfg.kind != "qNEI":
            raise IncompatibleAcquisitionFunctionError(
                "hybrid search spaces are served with qNoisyExpectedImprovement on the B200 engine "
                f"(got '{cfg.kind}')")
        if searchspace.continuous.has_interpoint_constraints or searchspace.continuous.constraints_lin_eq or \
                searchspace.continuous.constraints_lin_ineq:
            raise IncompatibilityError("continuous constraints are not supported by the B200 hybrid search")
        disc = searchspace.discrete.transform(candidates_exp)  # comp-rep of the discrete part, comes first
        cb = searchspace.continuous.comp_rep_bounds.to_numpy(dtype=np.float64)
        pend = None
        if pending is not None and len(pending) > 0:
            pend = searchspace.transform(pending, allow_extra=True).to_numpy(dtype=np.float64)
        pts, idx, value = recommend_hybrid(self._surrogate_model.device_gp, cfg, disc.to_numpy(dtype=np.float64), cb,
                                           batch_size, pend, self.n_mc_samples, _draw_sampler_seed())
        self._last_acq_values[:] = [value]
        rec_disc = searchspace.discrete.exp_rep.loc[disc.index[idx]]
        rec_cont = pd.DataFrame(pts[:, disc.shape[1]:], columns=searchspace.continuous.parameter_names,
                                index=rec_disc.index)
        return pd.concat([rec_disc, rec_cont], axis=1)

    def _recommend_discrete_without_subsets(self, subspace_discrete, candidates_exp, batch_size) -> pd.Index:
        cfg, searchspace, pending = self._context
        gp = self._scorer if self._scorer is not None else self._surrogate_model.device_gp
        return recommend_discrete_positions(gp, cfg, subspace_discrete, candidates_exp, batch_size, searchspace,
                                            pending, self.n_mc_samples, self._last_acq_values)

    def _recommend_discrete_with_subsets(self, subspace_discrete, candidates_exp, batch_size) -> pd.Index:
        """``recommend_discrete_with_subsets`` (botorch/discrete.py:21-75): optimise inside every feasible subset,
        keep the batch whose joint acquisition value is highest."""
        if subspace_discrete.n_subsets <= self.max_n_subsets:
            masks = subspace_discrete.subset_masks(candidates_exp, min_candidates=batch_size)
        else:
            masks = subspace_discrete.sample_subset_masks(candidates_exp, self.max_n_subsets,
                                                          min_candidates=batch_size)
        best_idxs, best_val = None, -np.inf
        for mask in masks:
            subset = candidates_exp.loc[mask]
            try:
                idxs = self._recommend_discrete_without_subsets(subspace_discrete, subset, batch_size)
            except InfeasibilityError:
                continue
            comp = subspace_discrete.transform(candidates_exp.loc[idxs])
            X = torch.from_numpy(comp.to_numpy(dtype=np.float64)).unsqueeze(0)
            val = float(self._botorch_acqf(X)[0])
            if val > best_val:
                best_idxs, best_val = idxs, val
        if best_idxs is None:
            raise InfeasibilityError(
                "No feasible solution could be found. Potentially the specified constraints are too restrictive.")
        return best_idxs

    # ---- diagnostics BayBE exposes through Campaign (bayesian/base.py:199-277) ---------------------------------
    def acquisition_values(self, candidates, searchspace, objective, measurements, pending_experiments=None,
                           acquisition_function=None) -> pd.Series:
        surrogate = self.get_surrogate(searchspace, objective, measurements)
        given = acquisition_function or self._get_acquisition_function(objective)
        acqf = mirror_acquisition_function(given)
        return acqf.evaluate(candidates, surrogate, searchspace, objective, measurements, pending_experiments,
                             jointly=False, **_integration_points(given, acqf, searchspace))

    def joint_acquisition_value(self, candidates, searchspace, objective, measurements, pending_experiments=None,
                                acquisition_function=None) -> float:
        surrogate = self.get_surrogate(searchspace, objective, measurements)
        given = acquisition_function or self._get_acquisition_function(objective)
        acqf = mirror_acquisition_function(given)
        return acqf.evaluate(candidates, surrogate, searchspace, objective, measurements, pending_experiments,
                             jointly=True, **_integration_points(given, acqf, searchspace))
