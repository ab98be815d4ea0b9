"""The interface of the scorers that run their own rounds on the device: ``HviScorer`` (qEHVI / qLogEHVI),
``ObjectiveScorer`` (non-affine objectives), ``NeiScorer`` (qNEI / qLogNEI), ``ParegoScorer`` (qLogNParEGO) and
``NehviScorer`` (qNEHVI).

A scorer defines ``values`` (scores, packed best key and a `report` map for every row of x, given the pending points,
the other points of a q-batch and the base samples) and ``n_sample_columns``; this base derives from them what the
recommenders and the acquisition callables use: ``base_samples``, ``round_best``, ``scores`` and ``joint_value``.
"""
from __future__ import annotations

import numpy as np
import torch

from baybe_b200 import _lib
from baybe_b200.engine import sobol_normal_samples

__all__ = ["Scorer"]


class Scorer:
    """Base of the scorers; subclasses set ``cfg`` and ``device`` and define ``values`` and ``n_sample_columns``."""

    def n_sample_columns(self, n_other: int) -> int | None:
        """Columns of the base samples of an evaluation with `n_other` pending and batch points (None: no samples)."""
        raise NotImplementedError

    def values(self, x, pend: np.ndarray | None, z: torch.Tensor | None, keep=None, index_offset: int = 0,
               want_scores: bool = True, batch: np.ndarray | None = None):
        """(scores or None, packed best key, report) for every row of x; `report` maps a value of the kernel (a
        float or an array) to the acquisition value."""
        raise NotImplementedError

    def base_samples(self, n_samples: int, n_other: int, seed: int) -> torch.Tensor | None:
        """Scrambled Sobol normals of ``n_sample_columns(n_other)`` dimensions (None where the scorer takes none)."""
        n = self.n_sample_columns(n_other)
        return None if n is None else sobol_normal_samples(n_samples, n, seed)

    def round_best(self, x, pend: np.ndarray, keep, index_offset: int, seed: int, n_samples: int):
        """One sequential-greedy round: (packed best key, report) -- see ``greedy_select``."""
        P = len(pend)
        _, key, report = self.values(x, pend if P else None, self.base_samples(n_samples, P, seed), keep,
                                     index_offset, want_scores=False)
        return key, report

    def scores(self, x, pend: np.ndarray | None, seed: int, n_samples: int,
               batch: np.ndarray | None = None) -> np.ndarray:
        """Acquisition value of every row given the pending points (and, for the scorers whose ``values`` takes
        them, the other points of its q-batch), float64."""
        P = 0 if pend is None else len(pend)
        Q = 0 if batch is None else len(batch)
        kw = {"batch": batch} if Q else {}
        s, _, report = self.values(x, pend if P else None, self.base_samples(n_samples, P + Q, seed), **kw)
        return report(s.double().cpu().numpy())

    def joint_value(self, rows, pend: np.ndarray | None, seed: int, n_samples: int) -> float:
        """Value of the q-batch `rows` given the pending points: the first row is the candidate, the other rows and
        the pending points are its pending points."""
        rows = np.asarray(rows, dtype=np.float64)
        rest = rows[1:] if pend is None else np.concatenate([rows[1:], np.asarray(pend, dtype=np.float64)], axis=0)
        if len(rest) > _lib.MAX_PENDING:
            raise NotImplementedError(f"joint evaluation supports at most {_lib.MAX_PENDING + 1} points")
        return float(self.scores(rows[:1], rest if len(rest) else None, seed, n_samples)[0])
