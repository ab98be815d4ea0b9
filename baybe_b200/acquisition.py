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
    "qNoisyExpectedHypervolumeImprovement", "qNEHVI", "qNegIntegratedPosteriorVariance", "qNIPV",
]


class IncompatibleAcquisitionFunctionError(Exception):
    """Same name/meaning as baybe.exceptions.IncompatibleAcquisitionFunctionError."""


def _space_kind(searchspace) -> str:
    return getattr(getattr(searchspace, "type", None), "name", "DISCRETE")


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

    def uses_scorer(self, objective, searchspace) -> bool:
        """True where ``scorer()`` (a ``baybe_b200.scoring.Scorer``) serves this spec on this objective and search
        space, False where the fused path does (``to_engine``)."""
        from baybe_b200.objectives import uses_objective_scorer

        return uses_objective_scorer(objective)

    def evaluate(self, candidates: pd.DataFrame, surrogate, searchspace, objective, measurements,
                 pending_experiments: pd.DataFrame | None = None, *, jointly: bool = False):
        """Acquisition values of the given candidates (acquisition/base.py:112-159)."""
        import torch

        from baybe_b200.engine import DEFAULT_MC_SAMPLES
        from baybe_b200.recommenders import _draw_sampler_seed, _scores_for

        if self.uses_scorer(objective, searchspace):
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

        kind = _space_kind(searchspace)
        if kind != "DISCRETE":
            raise IncompatibleAcquisitionFunctionError(
                f"'{type(objective).__name__}' with a non-affine objective is served on discrete search spaces only "
                f"by the B200 engine (got {kind})")
        surrogate.fit(searchspace, objective, measurements)
        flat = getattr(surrogate, "_surrogates_flat", None)
        gps = [s.device_gp for s in flat] if flat is not None else [surrogate.device_gp]
        return build_objective_scorer(self, gps, searchspace, objective, measurements)


def _evaluate_with_scorer(acqf, scorer, candidates: pd.DataFrame, searchspace, pending_experiments, jointly: bool):
    """``evaluate`` through a ``baybe_b200.scoring.Scorer``: one value per candidate, or the joint value of the batch
    [candidates; pending] (``Scorer.joint_value``)."""
    from baybe_b200.engine import DEFAULT_MC_SAMPLES
    from baybe_b200.recommenders import _draw_sampler_seed

    rows = searchspace.transform(candidates, allow_extra=True).to_numpy(dtype="float64")
    pend = None
    if pending_experiments is not None and len(pending_experiments) > 0:
        pend = searchspace.transform(pending_experiments, allow_extra=True).to_numpy(dtype="float64")
    seed = _draw_sampler_seed()
    if jointly:
        if len(rows) + (0 if pend is None else len(pend)) > 1 and not scorer.cfg.is_mc:
            raise IncompatibleAcquisitionFunctionError(
                f"'{type(acqf).__name__}' is analytic and cannot value a batch of {len(rows)} points jointly.")
        return scorer.joint_value(rows, pend, seed, DEFAULT_MC_SAMPLES)
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

    def uses_scorer(self, objective, searchspace) -> bool:
        """Discrete spaces: ``NeiScorer``; hybrid spaces: the fused path (``baybe_b200.hybrid``)."""
        return _space_kind(searchspace) == "DISCRETE" or super().uses_scorer(objective, searchspace)


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
class _ScoredAcquisitionFunction(AcquisitionFunction):
    """Specs for Pareto objectives that only a ``baybe_b200.scoring.Scorer`` serves (``scorer()``)."""

    supports_multi_output: ClassVar[bool] = True
    _scorer_module: ClassVar[str] = ""

    @staticmethod
    def compute_ref_point(array, maximize=None, factor: float = 0.1):
        from baybe_b200.multiobjective import compute_ref_point

        return compute_ref_point(array, maximize, factor)

    def uses_scorer(self, objective, searchspace) -> bool:
        return bool(getattr(objective, "is_multi_output", False))

    def to_engine(self, surrogate, searchspace, objective, measurements, pending_experiments=None) -> AcqConfig:
        raise IncompatibleAcquisitionFunctionError(
            f"'{type(self).__name__}' needs a multi-output objective; it is evaluated by "
            f"{self._scorer_module} (see scorer())")

    def evaluate(self, candidates: pd.DataFrame, surrogate, searchspace, objective, measurements,
                 pending_experiments: pd.DataFrame | None = None, *, jointly: bool = False):
        scorer = self.scorer(surrogate, searchspace, objective, measurements)
        return _evaluate_with_scorer(self, scorer, candidates, searchspace, pending_experiments, jointly)

    def _check_pareto(self, objective, searchspace, max_targets: int | None = None) -> None:
        """A multi-output objective on a discrete space and, with `max_targets`, 2 to `max_targets` affine targets
        (checked before the surrogate fit)."""
        from baybe_b200.multiobjective import _error, target_orientations

        if not getattr(objective, "is_multi_output", False):
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"'{type(self).__name__}' needs a multi-output (Pareto) objective")
        kind = _space_kind(searchspace)
        if kind != "DISCRETE":
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"'{type(self).__name__}' is served on discrete search spaces only by the B200 engine (got {kind})")
        if max_targets is None:
            return
        n_targets = len(objective.targets)
        if not 2 <= n_targets <= max_targets:
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"{self.abbreviation} on the B200 engine supports 2 to {max_targets} targets (got {n_targets})")
        target_orientations(objective)  # a target that is not affine raises here


@define(frozen=True)
class _ExpectedHypervolumeImprovement(_ScoredAcquisitionFunction):
    """acquisition/acqfs.py:342-418: Pareto objectives of 2 to 4 targets, scored by ``bb_hvi_score``
    (``baybe_b200.multiobjective``).  ``reference_point``: None (default factor 0.1), a factor, or coordinates in
    the oriented objective space; ``alpha``: None or 0.0 (exact partitioning)."""

    _scorer_module: ClassVar[str] = "baybe_b200.multiobjective.HviScorer"
    reference_point: float | tuple[float, ...] | None = field(default=None, converter=_reference_point)
    alpha: float | None = field(default=None, converter=lambda v: None if v is None else float(v))

    def scorer(self, surrogate, searchspace, objective, measurements):
        """Fit the per-target surrogates (a ``CompositeSurrogate``, surrogates/composite.py:96) and set up the
        reference point and the partitioning of the posterior-mean front."""
        from baybe_b200.multiobjective import build_hvi_scorer

        self._check_pareto(objective, searchspace)
        surrogate.fit(searchspace, objective, measurements)
        gps = [s.device_gp for s in surrogate._surrogates_flat]
        return build_hvi_scorer(self, gps, searchspace, objective, measurements)


@define(frozen=True)
class qExpectedHypervolumeImprovement(_ExpectedHypervolumeImprovement):
    """acquisition/acqfs.py:421-434."""

    abbreviation: ClassVar[str] = "qEHVI"


@define(frozen=True)
class qLogExpectedHypervolumeImprovement(_ExpectedHypervolumeImprovement):
    """acquisition/acqfs.py:437-451; tau_relu = 1e-6 and tau_max = 1e-2 as in ``AcqConfig``."""

    abbreviation: ClassVar[str] = "qLogEHVI"


@define(frozen=True)
class qLogNParEGO(_ScoredAcquisitionFunction):
    """acquisition/acqfs.py:328-336: Pareto objectives of 2 to 8 targets on discrete search spaces, scored by
    ``bb_parego_score`` (``baybe_b200.parego``): random simplex weights, augmented Chebyshev scalarisation of the
    normalised oriented targets and a qLogNEI of it over the measured rows, pruned as ``prune_baseline`` says (at
    most 31 points together with the pending points without pruning); tau_relu = 1e-6 and tau_max = 1e-2 as in
    ``AcqConfig``."""

    abbreviation: ClassVar[str] = "qLogNParEGO"
    _scorer_module: ClassVar[str] = "baybe_b200.parego.ParegoScorer"
    prune_baseline: bool = field(default=True, validator=instance_of(bool))

    def scorer(self, surrogate, searchspace, objective, measurements):
        """Check the objective and the space, fit the per-target surrogates (a ``CompositeSurrogate``), then draw
        the weights and set up the baseline and its pruning (``baybe_b200.parego.build_parego_scorer``)."""
        from baybe_b200.parego import build_parego_scorer

        self._check_pareto(objective, searchspace, _lib.PAREGO_MAX_TARGETS)
        surrogate.fit(searchspace, objective, measurements)
        gps = [s.device_gp for s in surrogate._surrogates_flat]
        return build_parego_scorer(self, gps, searchspace, objective, measurements)


@define(frozen=True)
class qNoisyExpectedHypervolumeImprovement(_ScoredAcquisitionFunction):
    """acquisition/acqfs.py:467-474: Pareto objectives of 2 to 4 targets on discrete search spaces
    (``baybe_b200.nehvi``): the improvement of a candidate over the sampled front of the measured rows, pruned as
    ``prune_baseline`` says (at most 31 points together with the pending points without pruning), one exact box
    decomposition per base sample (``bb_hvi_decompose``) and the hypervolume-improvement kernel ``bb_hvi_score``.
    ``reference_point``: None (default factor 0.1), a factor, or coordinates in the oriented objective space; the
    partitioning is always exact."""

    abbreviation: ClassVar[str] = "qNEHVI"
    _scorer_module: ClassVar[str] = "baybe_b200.nehvi.NehviScorer"
    reference_point: float | tuple[float, ...] | None = field(default=None, converter=_reference_point)
    prune_baseline: bool = field(default=True, validator=instance_of(bool))

    def scorer(self, surrogate, searchspace, objective, measurements):
        """Check the objective and the space, fit the per-target surrogates (a ``CompositeSurrogate``), then set up
        the reference point, the baseline and its pruning (``baybe_b200.nehvi.build_nehvi_scorer``)."""
        from baybe_b200.nehvi import build_nehvi_scorer

        self._check_pareto(objective, searchspace, _lib.HVI_MAX_TARGETS)
        surrogate.fit(searchspace, objective, measurements)
        gps = [s.device_gp for s in surrogate._surrogates_flat]
        return build_nehvi_scorer(self, gps, searchspace, objective, measurements)


def _incompatibility(msg: str) -> Exception:
    try:
        from baybe.exceptions import IncompatibilityError
    except ImportError:  # pragma: no cover - baybe absent
        return NotImplementedError(msg)
    return IncompatibilityError(msg)


def _positive_int_or_none(_, attr, value) -> None:
    if value is not None and (not isinstance(value, int) or isinstance(value, bool) or value <= 0):
        raise ValueError(f"'{attr.name}' must be a positive int or None (got {value!r})")


@define(frozen=True)
class qNegIntegratedPosteriorVariance(AcquisitionFunction):
    """acquisition/acqfs.py:28-138: global active learning on discrete search spaces (``baybe_b200.nipv``): the
    negative posterior variance averaged over integration points drawn from the whole discrete space, conditional on
    noisy observations of the candidate, the pending points and the other points of a q-batch (``bb_nipv_score``).
    Single targets without a transformation only; ``sampling_method``: "Random" (the plugin also takes BayBE's FPS
    points through the BayBE spec's ``get_integration_points``)."""

    abbreviation: ClassVar[str] = "qNIPV"
    sampling_n_points: int | None = field(default=None, validator=_positive_int_or_none)
    sampling_fraction: float | None = field(converter=lambda v: None if v is None else float(v))
    sampling_method: str = field(default="Random", converter=lambda v: str(getattr(v, "value", v)))

    @sampling_fraction.default
    def _default_sampling_fraction(self) -> float | None:
        return 1.0 if self.sampling_n_points is None else None

    @sampling_fraction.validator
    def _validate_sampling_fraction(self, attr, value) -> None:
        if value is not None and not 0.0 < value <= 1.0:
            raise ValueError(f"'{attr.name}' must be in (0, 1] (got {value})")
        if None not in (self.sampling_fraction, self.sampling_n_points):
            raise ValueError(
                f"For '{self.__class__.__name__}', the attributes '{attr.name}' and 'sampling_n_points' cannot "
                f"be specified at the same time.")

    def get_integration_points(self, searchspace) -> pd.DataFrame:
        """The integration rows of the discrete part (reference ``get_integration_points``, Random only)."""
        from baybe_b200.nipv import sample_integration_points

        return sample_integration_points(searchspace.discrete.comp_rep, self.sampling_n_points,
                                         self.sampling_fraction, self.sampling_method)

    def uses_scorer(self, objective, searchspace) -> bool:
        return True

    def evaluate(self, candidates: pd.DataFrame, surrogate, searchspace, objective, measurements,
                 pending_experiments: pd.DataFrame | None = None, *, jointly: bool = False, integration=None):
        """``AcquisitionFunction.evaluate`` with the integration points `integration` (comp-rep rows; None:
        ``get_integration_points``)."""
        if pending_experiments is not None and not self.supports_pending_experiments:  # pragma: no cover - q kind
            raise IncompatibleAcquisitionFunctionError("qNIPV does not support pending experiments")
        scorer = self.scorer(surrogate, searchspace, objective, measurements, integration=integration)
        return _evaluate_with_scorer(self, scorer, candidates, searchspace, pending_experiments, jointly)

    def to_engine(self, surrogate, searchspace, objective, measurements, pending_experiments=None) -> AcqConfig:
        raise IncompatibleAcquisitionFunctionError(
            "'qNegIntegratedPosteriorVariance' is evaluated by baybe_b200.nipv.NipvScorer (see scorer())")

    def scorer(self, surrogate, searchspace, objective, measurements, integration=None):
        """Check the objective and the space, fit the surrogate and send the integration points (`integration`, or
        ``get_integration_points``) to the device."""
        from baybe_b200.multiobjective import _error
        from baybe_b200.nipv import NipvScorer

        if getattr(objective, "is_multi_output", False):
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"'{type(self).__name__}' needs a single-target objective")
        if type(objective).__name__ == "DesirabilityObjective":
            raise _incompatibility(f"'{type(self).__name__}' currently supports single-target objectives only.")
        kind = _space_kind(searchspace)
        if kind != "DISCRETE":
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"'{type(self).__name__}' is served on discrete search spaces only by the B200 engine (got {kind})")
        targets = getattr(objective, "targets", None) or [getattr(objective, "_target", None)]
        tr = getattr(targets[0], "transformation", None)
        if tr is not None and type(tr).__name__ != "IdentityTransformation":
            raise _incompatibility(
                "'qNegIntegratedPosteriorVariance' currently does not support any target transformations.")
        surrogate.fit(searchspace, objective, measurements)
        if integration is None:
            integration = self.get_integration_points(searchspace)
        return NipvScorer(surrogate.device_gp, AcqConfig(kind="qNIPV"), integration.to_numpy(dtype="float64"))


qNIPV = qNegIntegratedPosteriorVariance
qNEI, qLogNEI = qNoisyExpectedImprovement, qLogNoisyExpectedImprovement
qNEHVI = qNoisyExpectedHypervolumeImprovement
qEHVI, qLogEHVI = qExpectedHypervolumeImprovement, qLogExpectedHypervolumeImprovement
PM, PSTD, qSR = PosteriorMean, PosteriorStandardDeviation, qSimpleRegret
EI, qEI, LogEI, qLogEI = ExpectedImprovement, qExpectedImprovement, LogExpectedImprovement, qLogExpectedImprovement
PI, qPI, UCB, qUCB = ProbabilityOfImprovement, qProbabilityOfImprovement, UpperConfidenceBound, qUpperConfidenceBound

_BY_NAME = {c.__name__: c for c in (PM, PSTD, qSR, EI, qEI, LogEI, qLogEI, PI, qPI, UCB, qUCB, qNEI, qLogNEI,
                                    qEHVI, qLogEHVI, qLogNParEGO, qNEHVI, qNIPV)}
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
