"""Acquisition-function specs with the reference's names, fields, abbreviations and class-level
flags (``/root/reference/baybe/acquisition/acqfs.py`` and ``acquisition/base.py:29-159``).
``to_botorch`` is replaced by ``to_engine`` (BoTorch is not part of this stack); ``evaluate`` has
the reference's signature and returns a ``pd.Series`` indexed like the candidates."""

from __future__ import annotations

from typing import ClassVar

import pandas as pd
from attrs import define, field
from attrs.validators import instance_of

from baybe_b200 import _lib
from baybe_b200.engine import AcqConfig

__all__ = [
    "AcquisitionFunction", "PosteriorMean", "PosteriorStandardDeviation", "qSimpleRegret",
    "ExpectedImprovement", "qExpectedImprovement", "LogExpectedImprovement",
    "qLogExpectedImprovement", "ProbabilityOfImprovement", "qProbabilityOfImprovement",
    "UpperConfidenceBound", "qUpperConfidenceBound", "convert_acqf",
    "PM", "PSTD", "qSR", "EI", "qEI", "LogEI", "qLogEI", "PI", "qPI", "UCB", "qUCB",
    "qNoisyExpectedImprovement", "qNEI", "qLogNoisyExpectedImprovement", "qLogNEI",
    "qExpectedHypervolumeImprovement", "qEHVI", "qLogExpectedHypervolumeImprovement", "qLogEHVI", "qLogNParEGO",
    "qNoisyExpectedHypervolumeImprovement", "qNEHVI",
]


class IncompatibleAcquisitionFunctionError(Exception):
    """Same name/meaning as baybe.exceptions.IncompatibleAcquisitionFunctionError."""


@define(frozen=True)
class AcquisitionFunction:
    """Base class (acquisition/base.py:29-54): flags derive from the leading ``q``."""

    abbreviation: ClassVar[str] = ""
    supports_multi_output: ClassVar[bool] = False

    @classmethod
    def _is_q(cls) -> bool:
        return cls.abbreviation.startswith("q")

    @property
    def is_analytic(self) -> bool:
        return not self._is_q()

    @property
    def supports_batching(self) -> bool:
        return self._is_q()

    @property
    def supports_pending_experiments(self) -> bool:
        return self._is_q()

    def _engine_kwargs(self) -> dict:
        return {}

    def to_engine(self, surrogate, searchspace, objective, measurements,
                  pending_experiments: pd.DataFrame | None = None) -> AcqConfig:
        """Counterpart of ``to_botorch`` (acquisition/base.py:61-84): resolve the context
        (objective orientation, best_f) into the engine's acquisition config."""
        from baybe_b200.objectives import uses_objective_scorer
        from baybe_b200.searchspace import objective_affine

        if pending_experiments is not None and not self.supports_pending_experiments:
            raise IncompatibleAcquisitionFunctionError(
                f"The chosen acquisition function of type '{type(self).__name__}' "
                f"does not support pending experiments.")
        if uses_objective_scorer(objective):
            raise IncompatibleAcquisitionFunctionError(
                f"'{type(objective).__name__}' is not affine in its targets; it is evaluated by "
                "baybe_b200.objectives.ObjectiveScorer (see scorer())")
        a, b, _ = objective_affine(objective)
        cfg = AcqConfig(kind=self.abbreviation, obj_scale=a, obj_shift=b, **self._engine_kwargs())
        if self.abbreviation in ("qLogEI", "qEI", "qPI", "EI", "LogEI", "PI"):
            # best_f = max_i o(mu(x_i)) over the training inputs (_builder.py:256-265)
            cfg = AcqConfig(kind=cfg.kind, best_f=surrogate.device_gp.best_f(cfg), beta=cfg.beta,
                            obj_scale=a, obj_shift=b, maximize=cfg.maximize)
        return cfg

    def evaluate(self, candidates: pd.DataFrame, surrogate, searchspace, objective, measurements,
                 pending_experiments: pd.DataFrame | None = None, *, jointly: bool = False):
        """Acquisition values of the given candidates (acquisition/base.py:112-159)."""
        import torch

        from baybe_b200.engine import DEFAULT_MC_SAMPLES
        from baybe_b200.objectives import uses_objective_scorer
        from baybe_b200.recommenders import _draw_sampler_seed, _scores_for

        if uses_objective_scorer(objective):
            if pending_experiments is not None and not self.supports_pending_experiments:
                raise IncompatibleAcquisitionFunctionError(
                    f"The chosen acquisition function of type '{type(self).__name__}' "
                    f"does not support pending experiments.")
            scorer = self.scorer(surrogate, searchspace, objective, measurements)
            return _evaluate_with_scorer(self, scorer, candidates, searchspace, pending_experiments, jointly)
        surrogate.fit(searchspace, objective, measurements)
        cfg = self.to_engine(surrogate, searchspace, objective, measurements, pending_experiments)
        comp = searchspace.transform(candidates, allow_extra=True)
        x = torch.from_numpy(comp.to_numpy(dtype="float64", copy=True))
        pend = None
        if pending_experiments is not None:
            pend = searchspace.transform(pending_experiments, allow_extra=True).to_numpy(dtype="float64")
        seed = _draw_sampler_seed()
        if jointly:
            # one q-batch [x_1..x_q ; X_pending] (botorch concatenates pending points behind the batch):
            # the joint kernel's "candidate first" order is exactly this order with x_1 as the candidate
            import numpy as np

            from baybe_b200.engine import sobol_normal_samples
            from baybe_b200._lib import MAX_PENDING

            rows = comp.to_numpy(dtype="float64")
            rest = rows[1:] if pend is None else np.concatenate([rows[1:], pend.reshape(-1, rows.shape[1])], axis=0)
            if len(rest) == 0:
                return float(_scores_for(surrogate.device_gp, cfg, x[:1], None, seed, DEFAULT_MC_SAMPLES)[0])
            if not cfg.is_mc:
                raise IncompatibleAcquisitionFunctionError(
                    f"'{type(self).__name__}' is analytic and cannot value a batch of {len(rows)} points jointly.")
            if len(rest) > MAX_PENDING:
                raise NotImplementedError(f"joint evaluation supports at most {MAX_PENDING + 1} points")
            z = sobol_normal_samples(DEFAULT_MC_SAMPLES, 1 + len(rest), seed)
            return float(surrogate.device_gp.score_joint(cfg, x[:1], rest, z)[0])
        scores = _scores_for(surrogate.device_gp, cfg, x, pend, seed, DEFAULT_MC_SAMPLES)
        return pd.Series(scores.double().cpu().numpy(), index=candidates.index)

    def scorer(self, surrogate, searchspace, objective, measurements):
        """Objectives that are not affine in their targets (desirability, non-affine single targets): fit the
        surrogate -- one model per target through a ``CompositeSurrogate`` for desirability -- and set up best_f
        and the compiled objective (``baybe_b200.objectives``)."""
        from baybe_b200.objectives import build_objective_scorer

        kind = getattr(getattr(searchspace, "type", None), "name", "DISCRETE")
        if kind != "DISCRETE":
            raise IncompatibleAcquisitionFunctionError(
                f"'{type(objective).__name__}' with a non-affine objective is served on discrete search spaces only "
                f"by the B200 engine (got {kind})")
        surrogate.fit(searchspace, objective, measurements)
        flat = getattr(surrogate, "_surrogates_flat", None)
        gps = [s.device_gp for s in flat] if flat is not None else [surrogate.device_gp]
        return build_objective_scorer(self, gps, searchspace, objective, measurements)


def _evaluate_with_scorer(acqf, scorer, candidates: pd.DataFrame, searchspace, pending_experiments, jointly: bool):
    """``evaluate`` through a scorer that runs its own rounds (``HviScorer``, ``ObjectiveScorer``): one value per
    candidate, or the joint value of the batch [candidates; pending] with the first candidate scored against the
    rest."""
    import numpy as np

    from baybe_b200._lib import MAX_PENDING
    from baybe_b200.engine import DEFAULT_MC_SAMPLES
    from baybe_b200.recommenders import _draw_sampler_seed

    rows = searchspace.transform(candidates, allow_extra=True).to_numpy(dtype="float64")
    pend = None
    if pending_experiments is not None and len(pending_experiments) > 0:
        pend = searchspace.transform(pending_experiments, allow_extra=True).to_numpy(dtype="float64")
    seed = _draw_sampler_seed()
    if jointly and hasattr(scorer, "joint_value"):  # the scorer tells batch points from pending points itself
        return scorer.joint_value(rows, pend, seed, DEFAULT_MC_SAMPLES)
    if jointly:  # candidate first, then the rest of the batch and the pending points
        rest = rows[1:] if pend is None else np.concatenate([rows[1:], pend], axis=0)
        if len(rest) and not scorer.cfg.is_mc:
            raise IncompatibleAcquisitionFunctionError(
                f"'{type(acqf).__name__}' is analytic and cannot value a batch of {len(rows)} points jointly.")
        if len(rest) > MAX_PENDING:
            raise NotImplementedError(f"joint evaluation supports at most {MAX_PENDING + 1} points")
        return float(scorer.scores(rows[:1], rest if len(rest) else None, seed, DEFAULT_MC_SAMPLES)[0])
    return pd.Series(scorer.scores(rows, pend, seed, DEFAULT_MC_SAMPLES), index=candidates.index)


@define(frozen=True)
class PosteriorMean(AcquisitionFunction):
    abbreviation: ClassVar[str] = "PM"


@define(frozen=True)
class PosteriorStandardDeviation(AcquisitionFunction):
    abbreviation: ClassVar[str] = "PSTD"
    maximize: bool = field(default=True, validator=instance_of(bool))

    def _engine_kwargs(self) -> dict:
        return {"maximize": self.maximize}


@define(frozen=True)
class qSimpleRegret(AcquisitionFunction):
    abbreviation: ClassVar[str] = "qSR"


@define(frozen=True)
class ExpectedImprovement(AcquisitionFunction):
    abbreviation: ClassVar[str] = "EI"


@define(frozen=True)
class qExpectedImprovement(AcquisitionFunction):
    abbreviation: ClassVar[str] = "qEI"


@define(frozen=True)
class LogExpectedImprovement(AcquisitionFunction):
    abbreviation: ClassVar[str] = "LogEI"


@define(frozen=True)
class qLogExpectedImprovement(AcquisitionFunction):
    abbreviation: ClassVar[str] = "qLogEI"


@define(frozen=True)
class ProbabilityOfImprovement(AcquisitionFunction):
    abbreviation: ClassVar[str] = "PI"


@define(frozen=True)
class qProbabilityOfImprovement(AcquisitionFunction):
    abbreviation: ClassVar[str] = "qPI"


@define(frozen=True)
class UpperConfidenceBound(AcquisitionFunction):
    abbreviation: ClassVar[str] = "UCB"
    beta: float = field(converter=float, default=0.2)

    def _engine_kwargs(self) -> dict:
        return {"beta": self.beta}


@define(frozen=True)
class qUpperConfidenceBound(AcquisitionFunction):
    abbreviation: ClassVar[str] = "qUCB"
    beta: float = field(converter=float, default=0.2)

    def _engine_kwargs(self) -> dict:
        return {"beta": self.beta}


def _space_kind(searchspace) -> str:
    return getattr(getattr(searchspace, "type", None), "name", "DISCRETE")


@define(frozen=True)
class _NoisyExpectedImprovement(AcquisitionFunction):
    """The noisy-EI family on discrete search spaces: ``baybe_b200.noisy.NeiScorer`` (``bb_nei_score``) with the
    measured rows as baseline, pruned to the points that are the best of at least one joint posterior sample
    (``prune_baseline=True``, the default) or kept whole (``prune_baseline=False``, at most 31 points together with
    the pending points)."""

    prune_baseline: bool = field(default=True, validator=instance_of(bool))

    def scorer(self, surrogate, searchspace, objective, measurements):
        """Check the objective, fit the surrogate, then set up the baseline and its pruning
        (``baybe_b200.noisy.build_nei_scorer``)."""
        from baybe_b200.noisy import build_nei_scorer

        kind = _space_kind(searchspace)
        if kind != "DISCRETE":
            raise IncompatibleAcquisitionFunctionError(
                f"'{type(self).__name__}' is scored by baybe_b200.noisy on discrete search spaces only (got {kind})")
        return build_nei_scorer(self, surrogate, searchspace, objective, measurements)

    def evaluate(self, candidates: pd.DataFrame, surrogate, searchspace, objective, measurements,
                 pending_experiments: pd.DataFrame | None = None, *, jointly: bool = False):
        if _space_kind(searchspace) != "DISCRETE":
            return super().evaluate(candidates, surrogate, searchspace, objective, measurements, pending_experiments,
                                    jointly=jointly)
        scorer = self.scorer(surrogate, searchspace, objective, measurements)
        return _evaluate_with_scorer(self, scorer, candidates, searchspace, pending_experiments, jointly)


@define(frozen=True)
class qNoisyExpectedImprovement(_NoisyExpectedImprovement):
    """acquisition/acqfs.py:226-232.  Discrete search spaces: ``baybe_b200.noisy``; hybrid search spaces:
    ``baybe_b200.hybrid``, which keeps every baseline point (its cost is one GEMM column each) and ignores
    ``prune_baseline``."""

    abbreviation: ClassVar[str] = "qNEI"


@define(frozen=True)
class qLogNoisyExpectedImprovement(_NoisyExpectedImprovement):
    """acquisition/acqfs.py:235-243; discrete search spaces only, tau_relu = 1e-6 and tau_max = 1e-2 as in
    ``AcqConfig``."""

    abbreviation: ClassVar[str] = "qLogNEI"


def _reference_point(v):
    if v is None:
        return None
    if isinstance(v, (int, float)):
        return float(v)
    return tuple(float(x) for x in v)


@define(frozen=True)
class _ExpectedHypervolumeImprovement(AcquisitionFunction):
    """acquisition/acqfs.py:342-418: Pareto objectives of 2 to 4 targets, scored by ``bb_hvi_score``
    (``baybe_b200.multiobjective``).  ``reference_point``: None (default factor 0.1), a factor, or coordinates in
    the oriented objective space; ``alpha``: None or 0.0 (exact partitioning)."""

    supports_multi_output: ClassVar[bool] = True
    reference_point: float | tuple[float, ...] | None = field(default=None, converter=_reference_point)
    alpha: float | None = field(default=None, converter=lambda v: None if v is None else float(v))

    @staticmethod
    def compute_ref_point(array, maximize=None, factor: float = 0.1):
        from baybe_b200.multiobjective import compute_ref_point

        return compute_ref_point(array, maximize, factor)

    def to_engine(self, surrogate, searchspace, objective, measurements, pending_experiments=None) -> AcqConfig:
        raise IncompatibleAcquisitionFunctionError(
            f"'{type(self).__name__}' needs a multi-output objective; it is evaluated by "
            "baybe_b200.multiobjective.HviScorer (see scorer())")

    def scorer(self, surrogate, searchspace, objective, measurements):
        """Fit the per-target surrogates (a ``CompositeSurrogate``, surrogates/composite.py:96) and set up the
        reference point and the partitioning of the posterior-mean front."""
        from baybe_b200.multiobjective import _error, build_hvi_scorer

        if not getattr(objective, "is_multi_output", False):
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"'{type(self).__name__}' needs a multi-output (Pareto) objective")
        kind = getattr(getattr(searchspace, "type", None), "name", "DISCRETE")
        if kind != "DISCRETE":
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"'{type(self).__name__}' is served on discrete search spaces only by the B200 engine (got {kind})")
        surrogate.fit(searchspace, objective, measurements)
        gps = [s.device_gp for s in surrogate._surrogates_flat]
        return build_hvi_scorer(self, gps, searchspace, objective, measurements)

    def evaluate(self, candidates: pd.DataFrame, surrogate, searchspace, objective, measurements,
                 pending_experiments: pd.DataFrame | None = None, *, jointly: bool = False):
        scorer = self.scorer(surrogate, searchspace, objective, measurements)
        return _evaluate_with_scorer(self, scorer, candidates, searchspace, pending_experiments, jointly)


@define(frozen=True)
class qExpectedHypervolumeImprovement(_ExpectedHypervolumeImprovement):
    """acquisition/acqfs.py:421-434."""

    abbreviation: ClassVar[str] = "qEHVI"


@define(frozen=True)
class qLogExpectedHypervolumeImprovement(_ExpectedHypervolumeImprovement):
    """acquisition/acqfs.py:437-451; tau_relu = 1e-6 and tau_max = 1e-2 as in ``AcqConfig``."""

    abbreviation: ClassVar[str] = "qLogEHVI"


@define(frozen=True)
class qLogNParEGO(AcquisitionFunction):
    """acquisition/acqfs.py:328-336: Pareto objectives of 2 to 8 targets on discrete search spaces, scored by
    ``bb_parego_score`` (``baybe_b200.parego``): random simplex weights, augmented Chebyshev scalarisation of the
    normalised oriented targets and a qLogNEI of it over the measured rows, pruned as ``prune_baseline`` says (at
    most 31 points together with the pending points without pruning); tau_relu = 1e-6 and tau_max = 1e-2 as in
    ``AcqConfig``."""

    abbreviation: ClassVar[str] = "qLogNParEGO"
    supports_multi_output: ClassVar[bool] = True
    prune_baseline: bool = field(default=True, validator=instance_of(bool))

    def to_engine(self, surrogate, searchspace, objective, measurements, pending_experiments=None) -> AcqConfig:
        raise IncompatibleAcquisitionFunctionError(
            f"'{type(self).__name__}' needs a multi-output objective; it is evaluated by "
            "baybe_b200.parego.ParegoScorer (see scorer())")

    def scorer(self, surrogate, searchspace, objective, measurements):
        """Check the objective and the space, fit the per-target surrogates (a ``CompositeSurrogate``), then draw
        the weights and set up the baseline and its pruning (``baybe_b200.parego.build_parego_scorer``)."""
        from baybe_b200.multiobjective import _error, target_orientations
        from baybe_b200.parego import build_parego_scorer

        if not getattr(objective, "is_multi_output", False):
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"'{type(self).__name__}' needs a multi-output (Pareto) objective")
        kind = _space_kind(searchspace)
        if kind != "DISCRETE":
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"'{type(self).__name__}' is served on discrete search spaces only by the B200 engine (got {kind})")
        n_targets = len(objective.targets)
        if not 2 <= n_targets <= _lib.PAREGO_MAX_TARGETS:
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"{self.abbreviation} on the B200 engine supports 2 to {_lib.PAREGO_MAX_TARGETS} targets "
                f"(got {n_targets})")
        target_orientations(objective)  # before the fit: a target that is not affine raises here
        surrogate.fit(searchspace, objective, measurements)
        gps = [s.device_gp for s in surrogate._surrogates_flat]
        return build_parego_scorer(self, gps, searchspace, objective, measurements)

    def evaluate(self, candidates: pd.DataFrame, surrogate, searchspace, objective, measurements,
                 pending_experiments: pd.DataFrame | None = None, *, jointly: bool = False):
        scorer = self.scorer(surrogate, searchspace, objective, measurements)
        return _evaluate_with_scorer(self, scorer, candidates, searchspace, pending_experiments, jointly)


@define(frozen=True)
class qNoisyExpectedHypervolumeImprovement(AcquisitionFunction):
    """acquisition/acqfs.py:467-474: Pareto objectives of 2 to 4 targets on discrete search spaces
    (``baybe_b200.nehvi``): the improvement of a candidate over the sampled front of the measured rows, pruned as
    ``prune_baseline`` says (at most 31 points together with the pending points without pruning), one exact box
    decomposition per base sample (``bb_hvi_decompose``) and the hypervolume-improvement kernel ``bb_hvi_score``.
    ``reference_point``: None (default factor 0.1), a factor, or coordinates in the oriented objective space; the
    partitioning is always exact."""

    abbreviation: ClassVar[str] = "qNEHVI"
    supports_multi_output: ClassVar[bool] = True
    reference_point: float | tuple[float, ...] | None = field(default=None, converter=_reference_point)
    prune_baseline: bool = field(default=True, validator=instance_of(bool))

    @staticmethod
    def compute_ref_point(array, maximize=None, factor: float = 0.1):
        from baybe_b200.multiobjective import compute_ref_point

        return compute_ref_point(array, maximize, factor)

    def to_engine(self, surrogate, searchspace, objective, measurements, pending_experiments=None) -> AcqConfig:
        raise IncompatibleAcquisitionFunctionError(
            f"'{type(self).__name__}' needs a multi-output objective; it is evaluated by "
            "baybe_b200.nehvi.NehviScorer (see scorer())")

    def scorer(self, surrogate, searchspace, objective, measurements):
        """Check the objective and the space, fit the per-target surrogates (a ``CompositeSurrogate``), then set up
        the reference point, the baseline and its pruning (``baybe_b200.nehvi.build_nehvi_scorer``)."""
        from baybe_b200.multiobjective import _error, target_orientations
        from baybe_b200.nehvi import build_nehvi_scorer

        if not getattr(objective, "is_multi_output", False):
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"'{type(self).__name__}' needs a multi-output (Pareto) objective")
        kind = _space_kind(searchspace)
        if kind != "DISCRETE":
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"'{type(self).__name__}' is served on discrete search spaces only by the B200 engine (got {kind})")
        n_targets = len(objective.targets)
        if not 2 <= n_targets <= _lib.HVI_MAX_TARGETS:
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"{self.abbreviation} on the B200 engine supports 2 to {_lib.HVI_MAX_TARGETS} targets "
                f"(got {n_targets})")
        target_orientations(objective)  # before the fit: a target that is not affine raises here
        surrogate.fit(searchspace, objective, measurements)
        gps = [s.device_gp for s in surrogate._surrogates_flat]
        return build_nehvi_scorer(self, gps, searchspace, objective, measurements)

    def evaluate(self, candidates: pd.DataFrame, surrogate, searchspace, objective, measurements,
                 pending_experiments: pd.DataFrame | None = None, *, jointly: bool = False):
        scorer = self.scorer(surrogate, searchspace, objective, measurements)
        return _evaluate_with_scorer(self, scorer, candidates, searchspace, pending_experiments, jointly)


qNEI, qLogNEI = qNoisyExpectedImprovement, qLogNoisyExpectedImprovement
qNEHVI = qNoisyExpectedHypervolumeImprovement
qEHVI, qLogEHVI = qExpectedHypervolumeImprovement, qLogExpectedHypervolumeImprovement
PM, PSTD, qSR = PosteriorMean, PosteriorStandardDeviation, qSimpleRegret
EI, qEI, LogEI, qLogEI = ExpectedImprovement, qExpectedImprovement, LogExpectedImprovement, qLogExpectedImprovement
PI, qPI, UCB, qUCB = ProbabilityOfImprovement, qProbabilityOfImprovement, UpperConfidenceBound, qUpperConfidenceBound

_BY_NAME = {c.__name__: c for c in (PM, PSTD, qSR, EI, qEI, LogEI, qLogEI, PI, qPI, UCB, qUCB, qNEI, qLogNEI,
                                    qEHVI, qLogEHVI, qLogNParEGO, qNEHVI)}
_BY_NAME.update({c.abbreviation: c for c in list(_BY_NAME.values())})


def convert_acqf(acqf) -> AcquisitionFunction:
    """String -> class lookup by name or abbreviation (acquisition/utils.py:21-23)."""
    if isinstance(acqf, AcquisitionFunction):
        return acqf
    try:
        return _BY_NAME[acqf]()
    except KeyError:
        raise ValueError(f"unknown or unsupported acquisition function {acqf!r}; the B200 engine "
                         f"implements {sorted(set(c.abbreviation for c in _BY_NAME.values()))}") from None
