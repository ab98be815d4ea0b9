"""Minimal stand-ins for the *input producers* of the hot path: parameters, the discrete
subspace (experimental vs computational representation), targets and the single-target
objective.  BayBE itself cannot be imported offline (cattrs/botorch missing), so tests and
examples use these; every class keeps the reference's attribute names and conventions so that a
real ``baybe.searchspace.SearchSpace`` / ``SingleTargetObjective`` can be passed to the
recommender and surrogate of this package unchanged (they are duck-typed on exactly these
attributes).  Nothing here is on the hot path.

Reference semantics mirrored (files under /root/reference/baybe):
  parameters/numerical.py:22,94        NumericalDiscreteParameter: comp value = the number itself
  parameters/categorical.py:35,65-83   CategoricalParameter: OHE (one column per label) or INT
  parameters/categorical.py:20-22,87-91 TaskParameter: INT code of the *sorted* label order
  searchspace/discrete.py:186,208      SubspaceDiscrete.from_product / from_dataframe
  searchspace/discrete.py:529-536      scaling bounds = per-parameter comp_df min/max
  searchspace/core.py:247-251,272-283  SearchSpace.scaling_bounds / task_idx / n_tasks
  objectives/single.py:66-91           SingleTargetObjective; minimize == negated objective
"""

from __future__ import annotations

import itertools
from typing import Sequence

import numpy as np
import pandas as pd
from attrs import define, field


@define(frozen=True)
class NumericalDiscreteParameter:
    name: str
    values: tuple = field(converter=lambda v: tuple(sorted(float(x) for x in v)))

    @property
    def comp_df(self) -> pd.DataFrame:
        return pd.DataFrame({self.name: list(self.values)}, index=pd.Index(self.values))

    @property
    def is_task(self) -> bool:
        return False


@define(frozen=True)
class CategoricalParameter:
    name: str
    values: tuple = field(converter=tuple)
    encoding: str = "OHE"

    @property
    def comp_df(self) -> pd.DataFrame:
        if self.encoding == "OHE":
            cols = [f"{self.name}_{v}" for v in self.values]
            return pd.DataFrame(np.eye(len(self.values)), columns=cols, index=pd.Index(self.values))
        if self.encoding == "INT":
            return pd.DataFrame({self.name: np.arange(len(self.values), dtype=float)},
                                index=pd.Index(self.values))
        raise ValueError(f"unknown encoding {self.encoding!r}")

    @property
    def is_task(self) -> bool:
        return False


@define(frozen=True)
class TaskParameter:
    name: str
    values: tuple = field(converter=lambda v: tuple(sorted(v)))
    active_values: tuple | None = None

    @property
    def comp_df(self) -> pd.DataFrame:
        return pd.DataFrame({self.name: np.arange(len(self.values), dtype=float)},
                            index=pd.Index(self.values))

    @property
    def is_task(self) -> bool:
        return True


Parameter = NumericalDiscreteParameter | CategoricalParameter | TaskParameter


@define
class SubspaceDiscrete:
    """exp_rep: one row per candidate in user units; comp_rep: the float64 encoding the model sees."""

    parameters: list
    exp_rep: pd.DataFrame
    comp_rep: pd.DataFrame = field(init=False)

    def __attrs_post_init__(self):
        if self.exp_rep.index.has_duplicates:
            raise ValueError("exp_rep index must be unique")
        self.comp_rep = self.transform(self.exp_rep)

    @classmethod
    def from_product(cls, parameters: Sequence[Parameter]) -> "SubspaceDiscrete":
        cols = [p.name for p in parameters]
        rows = list(itertools.product(*[p.values for p in parameters]))
        return cls(list(parameters), pd.DataFrame(rows, columns=cols))

    @classmethod
    def from_dataframe(cls, df: pd.DataFrame, parameters: Sequence[Parameter]) -> "SubspaceDiscrete":
        return cls(list(parameters), df[[p.name for p in parameters]].copy())

    def transform(self, df: pd.DataFrame, allow_extra: bool = True) -> pd.DataFrame:
        parts = []
        for p in self.parameters:
            comp = p.comp_df
            try:
                parts.append(comp.loc[df[p.name].to_numpy()].set_axis(df.index))
            except KeyError as e:
                raise ValueError(f"value of parameter {p.name!r} not in its allowed set: {e}") from e
        return pd.concat(parts, axis=1).astype(np.float64)

    def get_candidates(self) -> tuple[pd.DataFrame, pd.DataFrame]:
        return self.exp_rep, self.comp_rep

    @property
    def scaling_bounds(self) -> pd.DataFrame:
        mins, maxs = [], []
        for p in self.parameters:
            c = p.comp_df
            mins.append(c.min())
            maxs.append(c.max())
        return pd.DataFrame([pd.concat(mins), pd.concat(maxs)], index=["min", "max"])

    @property
    def n_subsets(self) -> int:
        return 0


@define
class SearchSpace:
    discrete: SubspaceDiscrete

    @classmethod
    def from_product(cls, parameters: Sequence[Parameter]) -> "SearchSpace":
        return cls(SubspaceDiscrete.from_product(parameters))

    @classmethod
    def from_dataframe(cls, df: pd.DataFrame, parameters: Sequence[Parameter]) -> "SearchSpace":
        return cls(SubspaceDiscrete.from_dataframe(df, parameters))

    @property
    def parameters(self) -> tuple:
        return tuple(self.discrete.parameters)

    @property
    def comp_rep_columns(self) -> tuple[str, ...]:
        return tuple(self.discrete.comp_rep.columns)

    @property
    def scaling_bounds(self) -> pd.DataFrame:
        return self.discrete.scaling_bounds

    @property
    def task_idx(self) -> int | None:
        for p in self.parameters:
            if p.is_task:
                return self.comp_rep_columns.index(p.name)
        return None

    @property
    def n_tasks(self) -> int:
        for p in self.parameters:
            if p.is_task:
                return len(p.values)
        return 1

    def transform(self, df: pd.DataFrame, allow_extra: bool = True) -> pd.DataFrame:
        return self.discrete.transform(df, allow_extra=allow_extra)


@define(frozen=True)
class NumericalTarget:
    name: str
    minimize: bool = False


@define(frozen=True)
class SingleTargetObjective:
    """o(y) = y for maximisation, -y for minimisation (the affine case the engine supports)."""

    target: NumericalTarget

    @property
    def targets(self) -> tuple:
        return (self.target,)

    @property
    def is_multi_output(self) -> bool:
        return False


def objective_affine(objective) -> tuple[float, float, str]:
    """(scale a, shift b, target name) of the oriented single-target objective o = a*y + b.

    Accepts this module's SingleTargetObjective or a real BayBE one whose target carries an
    Identity/Affine transformation (objectives/single.py:77-91); anything else is rejected like
    the reference rejects non-affine chains for analytic acquisition functions."""
    targets = getattr(objective, "targets", None)
    if targets is None or len(targets) != 1:
        raise NotImplementedError("only single-target objectives are supported by the B200 engine")
    a, b = target_affine(targets[0])
    return a, b, targets[0].name


def target_affine(t) -> tuple[float, float]:
    """(a, b) of one target oriented for maximisation, o = a*y + b (Identity/Affine transformations only)."""
    a, b = 1.0, 0.0
    tr = getattr(t, "transformation", None)
    if tr is not None:
        name = type(tr).__name__
        if name == "AffineTransformation":
            a, b = float(tr.factor), float(tr.shift)
        elif name != "IdentityTransformation":
            raise NotImplementedError(
                f"target transformation {name} is not affine; fall back to the reference path")
    if getattr(t, "minimize", False):
        a, b = -a, -b
    return a, b
