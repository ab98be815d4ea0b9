"""The float64 training-side caches every scorer relies on, checked at float64 precision at every Cholesky block
boundary up to BB_MAX_TRAIN = 1024 training points:

  a. bb_model_build's blocked Cholesky (k_chol_diag / _trsm / _update) and blocked triangular inverse (k_trinv_diag /
     _offdiag): elementwise a-priori backward-error bounds, which need no condition number;
  b. alpha (k_alpha), its fp32 copy, linv32 and the fp16 hi/lo tensor-core image of L^-1 (k_build_rimg);
  c. the model scalars against oracle.build_model;
  d. bb_joint_posterior and bb_pending_stats (k_pending_w, k_pending_cov) against oracle.posterior_joint;
  e. the MAP-fit objectives bb_fit_eval / bb_fit_eval_loo against float64 autograd (tests/helpers.py::HostMLL);
  f. the jitter escalation of bb_model_build (0, 1e-8, 1e-7, 1e-6, then BB_ERR_NOT_PD) against the oracle's
     _psd_safe_cholesky;
  g. the pending-point statistics of a 4096-bit fingerprint model at n = 1024, whose k_pending_w launch needs more
     than the default 48 KB of shared memory.

The device arrays are read straight from the model blob (gp._blob).  The Cholesky factor itself is not exported: it is
left in place in the blob's Gram-matrix slot, the next array after linv32 in make_layout (model.cu); every row checks
that its diagonal is exactly the reciprocal of the diagonal of the exported L^-1, so a change of the layout fails
loudly instead of comparing the wrong memory.

Bounds, with u = 2^-53 and gamma_k = k u / (1 - k u); each row prints its worst err/bound per check:

  a. L: |L L^T - K| <= c (gamma_{n+1} |L||L^T| + dK), c = 2 (Higham, Accuracy and Stability of Numerical Algorithms,
     Thm 10.3, for any order of the inner products, blocked included; the second unit of c covers the host's own
     product).  K is restated on the host from the device's normalised inputs with the device's formula (direct
     differences summed in column order); dK = 4 u (d + 8)(1 + r2_ij) |K_ij| off the diagonal (0 on it) bounds the
     difference of two float64 evaluations of the kernel (r2 to gamma_{d+5} relative each, a relative slope
     |d ln k / d ln r2| <= 1.2 (1 + r2), a few units in exp and the polynomial).
     X = L^-1: |L X - I| <= c (gamma_n |L||X| + 2 gamma_32 |L_D||X_D||L_D||X|), c = 2.  k_trinv_diag is column-wise
     forward substitution (right residual within gamma_32 |L||X|, Higham ch. 14); k_trinv_offdiag forms
     X_IJ = -X_II (sum_K L_IK X_KJ), whose right residual adds the diagonal-block term (L_D, X_D: the 32 x 32 diagonal
     blocks).  The left residual |X L - I| carries the factor's conditioning for this method and is not bounded a
     priori; the oracle's own Cholesky differs from the device's by a forward error that does, so both bounds use
     the device's factor.
  b. alpha: |alpha - X^T (X r)| <= c gamma_n |X|^T |X||r|, c = 4 (two triangular products on the device and two on
     the host).  Residual: |K alpha - r| <= c n u (|K||alpha| + |r|), c = 4.  This one is empirical, not a priori:
     alpha comes from the explicit inverse, whose residual may carry cond(L); measured on an H100 (700 W) at 1.25 for
     n = 1 and at most 0.41 from n = 2 on, up to cond(K) ~ 2e6.  alpha32, linv32: exact fp32 roundings of the float64
     arrays.
     rimg: |hi + lo - s L^-1| <= c (2^-22 |s L^-1| + 2^-25), c = 2 (fp16 split of the fp32-rounded value: 2^-11 twice,
     the subnormal spacing 2^-24 halved).
  c. y_mean, y_std: |dev - oracle| <= 2^-24 |oracle| + 4 n u max(1, max|y|) (fp32 rounding and two summation
     orders); prior_scale, jitter and jitter_tries exact.
  d. |dmu| <= c u (n kappa + d + A2) y_std (1 + sum|alpha| k_max), |dcov| <= c u (n kappa + d + A2) y_std^2 k_max,
     |dbeta| <= 2^-24 |beta| + c u (n kappa + d + A2) max|beta|, c = 8 (measured on an H100 (700 W): mu 5.8e-4, cov
     8.6e-3 of these bounds at worst; beta 0.98, where its fp32 rounding term dominates):
     kappa = cond(K) from the oracle's factor, A2 the largest squared norm of a centred, lengthscale-scaled row (the
     oracle's |a|^2 + |b|^2 - 2 a.b distance cancels to u A2), k_max the largest prior variance.  The oracle is fed
     the device's fp32 inputs (rows, bounds, y statistics, mean constant) like test_gpu_nei.py.  fp32 outputs equal
     the rounded float64 ones exactly.  Matern-1/2 rows stay out of this check: near coincident rows the oracle's
     u A2 in r^2 becomes sqrt(u A2) ~ 1e-8 in k = exp(-r), an fp32-sized error of the oracle itself.
  e. |dvalue| <= c n u kappa max(1, |value|), |dgrad|_inf <= c n u kappa max(1, |grad|_inf), kappa = cond(K) of the
     fit's Gram matrix from the oracle, theta's noise >= 1e-3; c = 1 (measured on an H100 (700 W) at 0.0077 at worst,
     n = 33, up to kappa = 7e4).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import pytest
import torch

import oracle
from baybe_b200.synthetic import PRIOR_MODE_NOISE, Workload, fingerprint_workload, prior_mode_lengthscale, smooth_target
from tests.helpers import HostMLL, oracle_model

U = 2.0 ** -53
EPS32 = 2.0 ** -24
KCHUNK, KNB, MAX_TRAIN = 64, 32, 1024
RESIDENT_TRAIN_BYTES = 56 * 1024


def gamma(k: int) -> float:
    return k * U / (1.0 - k * U)


def layout(n: int, d: int) -> dict:
    """Block count, ragged last block, n_pad and the wide switch of n training points in d columns, as make_layout
    (model.cu) and launch_cholesky compute them."""
    n_pad = (n + KCHUNK - 1) // KCHUNK * KCHUNK
    d_pad = (d + 3) // 4 * 4
    return dict(nb=(n + KNB - 1) // KNB, ragged=n % KNB != 0, n_pad=n_pad,
                wide=n_pad * d_pad * 4 > RESIDENT_TRAIN_BYTES or n_pad > 512)


# ------------------------------------------------------------------------------------------
# the shape table
# ------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Row:
    n: int
    family: str
    d: int = 6  # numeric columns (a task column comes on top)
    outputscale: float | None = None
    ard: bool = False  # ARD lengthscales over 0.3-3 times the prior mode, the last numeric column inactive
    tasks: int = 1
    degenerate: bool = False  # first numeric column with upper == lower
    const_y: bool = False
    noise: float = PRIOR_MODE_NOISE
    joint: bool = False  # also check bb_joint_posterior / bb_pending_stats (d)

    @property
    def name(self) -> str:
        tags = [f"n{self.n}", self.family, f"d{self.d}"]
        tags += [f"os{self.outputscale}"] * (self.outputscale is not None) + ["ard"] * self.ard
        tags += [f"T{self.tasks}"] * (self.tasks > 1) + ["degen"] * self.degenerate + ["consty"] * self.const_y
        return "_".join(tags + [f"noise{self.noise:.0e}"] * (self.noise != PRIOR_MODE_NOISE))

    def width(self) -> int:
        return self.d + (self.tasks > 1)


M12, M32, M52, RBF = "matern12", "matern32", "matern52", "rbf"

# n crosses every 32-row Cholesky block count (nb = 1..32) with full and ragged last blocks, every 64-row n_pad from
# 64 to 1024 and both wide states (n_pad > 512, or n_pad * d_pad * 4 > 56 KB at d = 120).  Families, output scale,
# ARD with an inactive column, task kernels (T = 2, 4, 16), a degenerate range, n = 1 and a constant target are
# spread over the rows.
SHAPES = [
    Row(1, M52),
    Row(2, RBF, outputscale=2.0),
    Row(31, M32, ard=True, joint=True),
    Row(32, M12, tasks=2),
    Row(33, M52, const_y=True, joint=True),
    Row(63, RBF, degenerate=True),
    Row(64, M32, outputscale=0.5, tasks=4),
    Row(65, M52, noise=1e-4),
    Row(96, M12, ard=True),
    Row(97, RBF, d=120),
    Row(129, M32, tasks=16, joint=True),
    Row(192, M52, outputscale=1.5),
    Row(200, RBF, ard=True, degenerate=True),
    Row(255, M12),
    Row(256, M32, tasks=4, ard=True, joint=True),
    Row(257, M52),
    Row(320, RBF, tasks=2),
    Row(330, M12, outputscale=3.0),
    Row(384, M32, noise=1e-4),
    Row(400, M52, tasks=16),
    Row(448, RBF, ard=True),
    Row(470, M12),
    Row(511, M32, degenerate=True),
    Row(512, M52, outputscale=0.7),
    Row(513, RBF, joint=True),
    Row(576, M12, tasks=4),
    Row(600, M32, ard=True),
    Row(640, M52, tasks=2, outputscale=1.2),
    Row(650, RBF),
    Row(704, M12, noise=1e-4),
    Row(710, M32, tasks=16),
    Row(767, M52, ard=True),
    Row(800, RBF, outputscale=2.5),
    Row(820, M12),
    Row(864, M32, tasks=4),
    Row(890, M52),
    Row(928, RBF, degenerate=True, ard=True),
    Row(950, M12, outputscale=0.4),
    Row(992, M32),
    Row(1000, M52, tasks=16, joint=True),
    Row(1023, RBF, noise=1e-4, joint=True),
    Row(1024, M12, tasks=2),
]


def workload(row: Row, n_query: int = 0) -> Workload:
    """Training data of a row in raw units: random bounds, rows drawn inside them, a smooth target; `n_query`
    further rows inside the bounds as the workload's candidates."""
    rng = np.random.default_rng(1000 + row.n)
    d = row.d
    lo = rng.uniform(-2.0, 1.0, d)
    hi = lo + rng.uniform(0.5, 3.0, d)
    if row.degenerate:
        hi[0] = lo[0]
    draw = lambda m: lo + (hi - lo) * rng.random((m, d))  # noqa: E731
    x, q = draw(row.n), draw(n_query)
    y = np.full(row.n, 3.7) if row.const_y else smooth_target((x - lo) / np.where(hi > lo, hi - lo, 1.0))
    y = y + (0.0 if row.const_y else 0.01 * rng.standard_normal(row.n))
    ls = np.full(d, prior_mode_lengthscale(d))
    if row.ard:
        ls = ls * np.linspace(0.3, 3.0, d)
        ls[-1] = -1.0
    T = row.tasks
    task_col = task_covar = None
    noise, mean_const = np.array([row.noise]), np.array([0.1])
    if T > 1:
        x = np.concatenate([x, (np.arange(row.n) % T)[:, None].astype(np.float64)], axis=1)
        q = np.concatenate([q, rng.integers(0, T, (n_query, 1)).astype(np.float64)], axis=1)
        lo, hi, ls = np.append(lo, 0.0), np.append(hi, T - 1.0), np.append(ls, -1.0)
        W = rng.uniform(0.2, 1.0, (T, T))
        task_covar = W @ W.T + np.diag(rng.uniform(0.05, 0.3, T))
        task_covar /= task_covar.max()
        task_col = d
        noise = row.noise * rng.uniform(1.0, 2.0, T)
        mean_const = rng.normal(0.0, 0.2, T)
    return Workload(name=row.name, candidates=q, train_idx=np.arange(0), train_x=x, train_y=y,
                    bounds=np.stack([lo, hi]), family=row.family, lengthscale=ls, noise=noise,
                    mean_const=mean_const, outputscale=row.outputscale, task_col=task_col, task_covar=task_covar)


# ------------------------------------------------------------------------------------------
# CPU: the table's reach and the premise of the jitter construction
# ------------------------------------------------------------------------------------------
def test_shapes_reach_every_block_count_and_n_pad():
    lay = [layout(r.n, r.width()) for r in SHAPES]
    assert {x["nb"] for x in lay} == set(range(1, MAX_TRAIN // KNB + 1))
    assert {x["ragged"] for x in lay} == {True, False}
    assert {x["ragged"] for x in lay if x["nb"] == MAX_TRAIN // KNB} == {True, False}  # the last block at n_pad 1024
    assert {x["n_pad"] for x in lay} == set(range(KCHUNK, MAX_TRAIN + 1, KCHUNK))
    assert {x["wide"] for x in lay} == {True, False}
    assert any(x["wide"] and x["n_pad"] <= 512 for x in lay)  # wide by its features alone
    assert {r.family for r in SHAPES} == {M12, M32, M52, RBF}
    assert {r.tasks for r in SHAPES} >= {1, 2, 4, 16}
    assert any(r.ard for r in SHAPES) and any(r.outputscale for r in SHAPES) and any(r.degenerate for r in SHAPES)
    assert any(r.const_y for r in SHAPES) and any(r.n == 1 for r in SHAPES)
    assert any(r.joint and r.tasks > 1 for r in SHAPES) and any(r.joint and layout(r.n, r.width())["wide"]
                                                               for r in SHAPES)
    assert {layout(r.n, r.width())["n_pad"] for r in SHAPES if r.joint} >= {64, 1024}
    assert not any(r.joint and r.family == M12 for r in SHAPES)  # see the module docstring, d.


# Jitter construction: all training rows at one numeric point, n_t rows per task, so that K = B[t_i, t_j] + 1e-4 I
# (noise at the floor).  With B = [[a, b], [b, a]], a - b = -(1e-4 + delta) / n_t, a + b = 1, the smallest
# eigenvalue of K is -delta.  delta sits halfway between consecutive jitter steps (float64 roundoff of K's eigenvalues
# is ~1e-14 here), so the step psd_safe_cholesky stops at is fixed.
JITTER_NT = 40
JITTER_CASES = {  # delta -> (jitter_tries, jitter); None: not positive definite after 1e-6
    -5e-9: (0, 0.0),
    5e-9: (1, 1e-8),
    5.5e-8: (2, 1e-8 * 10),
    5.5e-7: (3, 1e-8 * 100),
    5e-6: None,
}


def jitter_model(delta: float, nt: int = JITTER_NT) -> dict:
    lam = -(1e-4 + delta) / nt
    B = np.array([[(1.0 + lam) / 2, (1.0 - lam) / 2], [(1.0 - lam) / 2, (1.0 + lam) / 2]])
    x = np.stack([np.full(2 * nt, 0.5), np.arange(2 * nt) % 2], axis=1).astype(np.float64)
    y = np.random.default_rng(5).standard_normal(2 * nt)
    return dict(train_x=x, train_y=y, bounds=np.array([[0.0, 0.0], [1.0, 1.0]]), family=RBF,
                lengthscale=np.array([0.7, -1.0]), noise=np.array([1e-4, 1e-4]), mean_const=np.zeros(2),
                outputscale=None, task_col=1, task_covar=B)


def _oracle_jitter_model(kw):
    spec = oracle.KernelSpec(family=kw["family"], lengthscale=kw["lengthscale"][:1], active_dims=[0],
                             task_idx=1, task_covar=kw["task_covar"])
    return oracle.build_model(spec, kw["train_x"], kw["train_y"], kw["bounds"], noise=kw["noise"],
                              mean_const=kw["mean_const"])


@pytest.mark.parametrize("delta", list(JITTER_CASES))
def test_jitter_construction_needs_its_intended_jitter(delta):
    kw = jitter_model(delta)
    n = len(kw["train_y"])
    tid = kw["train_x"][:, 1].astype(int)
    K = torch.as_tensor(kw["task_covar"][tid][:, tid] + 1e-4 * np.eye(n))
    assert abs(float(torch.linalg.eigvalsh(K)[0]) + delta) <= 1e-12
    want = JITTER_CASES[delta]
    if want is None:
        with pytest.raises(RuntimeError):
            oracle.reference_path._psd_safe_cholesky(K)
        with pytest.raises(RuntimeError):
            _oracle_jitter_model(kw)
    else:
        _, jit = oracle.reference_path._psd_safe_cholesky(K)
        assert jit == want[1]
        assert _oracle_jitter_model(kw).jitter == want[1]


def test_pending_shared_memory_of_a_4096_bit_model_needs_the_opt_in():
    """k_pending_w's 8 (d + 2n) dynamic bytes plus its 2 KB static reduction buffer exceed the default 48 KB launch
    limit at d = 4096, n = 1024 (so (g) needs the opt-in), and stay below the H100's 227 KB opt-in limit."""
    need = 8 * (4096 + 2 * 1024) + 8 * 256
    assert need == 51200 and need > 48 * 1024 and need <= 227 * 1024


# ------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------
def blob(gp, ptr: int, count: int, dtype) -> np.ndarray:
    """`count` elements of `dtype` at device pointer `ptr` inside gp's model blob."""
    off = int(ptr) - gp._blob.data_ptr()
    nbytes = count * np.dtype(dtype).itemsize
    assert 0 <= off and off + nbytes <= gp._blob.numel()
    return gp._blob[off:off + nbytes].cpu().numpy().view(dtype)


def device_arrays(gp) -> dict:
    m = gp.model
    n, n_pad, d = m.n, m.n_pad, m.d
    kmat = m.d_linv32 + 4 * n_pad * n_pad  # make_layout: the Gram matrix slot follows linv32 (1024-aligned already)
    resid = kmat + (8 * n * n + 1023) // 1024 * 1024
    n_tiles = m.n_chunks * (m.n_chunks + 1) // 2
    return dict(
        X=blob(gp, m.d_linv, n * n, np.float64).reshape(n, n),
        L=blob(gp, kmat, n * n, np.float64).reshape(n, n),
        r=blob(gp, resid, n, np.float64),
        xn=blob(gp, m.d_xn64, n * d, np.float64).reshape(n, d),
        alpha64=blob(gp, m.d_alpha64, n, np.float64),
        alpha32=blob(gp, m.d_alpha, n_pad, np.float32),
        linv32=blob(gp, m.d_linv32, n_pad * n_pad, np.float32).reshape(n_pad, n_pad),
        rimg=blob(gp, m.d_rimg, n_tiles * 16384, np.uint8),
    )


def host_gram(xn: np.ndarray, w: Workload, prior_scale: float, jitter: float) -> tuple[np.ndarray, np.ndarray]:
    """(K + noise + jitter, bound on the difference of two float64 evaluations of it) with the device's formula."""
    n, d = xn.shape
    T = 1 if w.task_covar is None else w.task_covar.shape[0]
    inv_ls = np.array([0.0 if (j == w.task_col or not w.lengthscale[j] > 0) else 1.0 / w.lengthscale[j]
                       for j in range(d)])
    r2 = np.zeros((n, n))
    for j in range(d):
        if inv_ls[j] != 0.0:
            u = (xn[:, None, j] - xn[None, :, j]) * inv_ls[j]
            r2 += u * u
    if w.family == RBF:
        k = np.exp(-0.5 * r2)
    else:
        r = np.sqrt(np.maximum(r2, 1e-30))
        if w.family == M12:
            k = np.exp(-r)
        elif w.family == M32:
            s = 1.7320508075688772 * r
            k = (1.0 + s) * np.exp(-s)
        else:
            s = 2.23606797749979 * r
            k = (1.0 + s + (5.0 / 3.0) * r2) * np.exp(-s)
    np.fill_diagonal(k, 1.0)
    tid = np.zeros(n, dtype=int) if w.task_col is None else np.rint(xn[:, w.task_col]).astype(int)
    tcov = prior_scale * (np.ones((1, 1)) if w.task_covar is None else w.task_covar)
    K = k * tcov[tid][:, tid]
    noise = np.maximum(np.broadcast_to(w.noise, (T,))[tid], 1e-4)
    K[np.diag_indices(n)] += noise + jitter
    dK = 4.0 * U * (d + 8) * (1.0 + r2) * np.abs(K)
    np.fill_diagonal(dK, 0.0)
    return K, dK


def inverse_bound(L: np.ndarray, X: np.ndarray) -> np.ndarray:
    """gamma_n |L||X| + 2 gamma_32 |L_D||X_D||L_D||X| (see the module docstring)."""
    n = L.shape[0]
    aL, aX = np.abs(L), np.abs(X)
    out = gamma(n) * (aL @ aX)
    for b in range(0, n, KNB):
        s = slice(b, min(b + KNB, n))
        P = aL[s, s] @ aX[s, s] @ aL[s, s]
        out[s] += 2 * gamma(KNB) * (P @ aX[s])
    return out


def rimg_index() -> np.ndarray:
    """fp16 element index of (row r, k column kk) inside one 64 x 64 128-byte-swizzled panel (sw128_offset)."""
    r, kk = np.meshgrid(np.arange(64), np.arange(64), indexing="ij")
    return r * 64 + (((kk >> 3) ^ (r & 7)) << 3) + (kk & 7)


def decode_rimg(raw: np.ndarray, n_chunks: int) -> np.ndarray:
    """hi + lo of every tile, placed at [j = 64 s + r, i = 64 c + kk] of an n_pad x n_pad matrix (float64)."""
    idx = rimg_index()
    out = np.zeros((64 * n_chunks, 64 * n_chunks))
    t = 0
    for c in range(n_chunks):
        for s in range(c, n_chunks):
            tile = raw[t * 16384:(t + 1) * 16384]
            hi = tile[:8192].view(np.float16).astype(np.float64)[idx]
            lo = tile[8192:].view(np.float16).astype(np.float64)[idx]
            out[64 * s:64 * s + 64, 64 * c:64 * c + 64] = hi + lo
            t += 1
    return out


def _report(name: str, **ratios):
    print(f"[{name}] " + " ".join(f"{k}={v:.3g}" for k, v in ratios.items()))


def _ratio(err: np.ndarray, bound: np.ndarray) -> float:
    return float(np.max(err / np.maximum(bound, np.finfo(np.float64).tiny))) if err.size else 0.0


JITTER_STEPS = {0.0: 0, 1e-8: 1, 1e-8 * 10: 2, 1e-8 * 100: 3}


# ------------------------------------------------------------------------------------------
# GPU: a, b, c per row
# ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("row", SHAPES, ids=lambda r: r.name)
def test_model_build_float64(row, cuda_device):
    from baybe_b200 import DeviceGP

    w = workload(row)
    gp = DeviceGP(device=cuda_device, **w.gp_kwargs())
    m = gp.model
    n, d = row.n, w.train_x.shape[1]
    lay = layout(n, d)
    assert (m.n, m.n_pad, bool(m.wide)) == (n, lay["n_pad"], lay["wide"])
    om = oracle_model(w)
    a = device_arrays(gp)
    X, L = a["X"], a["L"]

    # c. scalars
    y = w.train_y
    ytol = 4 * n * U * max(1.0, float(np.abs(y).max()))
    assert abs(m.y_mean - om.y_mean) <= EPS32 * abs(om.y_mean) + ytol, (m.y_mean, om.y_mean)
    assert abs(m.y_std - om.y_std) <= EPS32 * abs(om.y_std) + ytol, (m.y_std, om.y_std)
    if n == 1 or row.const_y:
        assert m.y_std == 1.0
    assert m.prior_scale == np.float32(row.outputscale or 1.0)
    assert m.jitter == om.jitter and m.jitter_tries == JITTER_STEPS[om.jitter]

    # a. the factor and its inverse
    assert np.array_equal(np.triu(L, 1), np.zeros_like(L)) and np.array_equal(np.triu(X, 1), np.zeros_like(X))
    assert np.array_equal(np.diag(X), 1.0 / np.diag(L)), "the Gram-matrix slot of the blob does not hold L"
    # normalised training rows: (x - lower) * (1 / range), range 1 where degenerate, the task column raw
    rng = w.bounds[1] - w.bounds[0]
    inv_range = 1.0 / np.where(np.abs(rng) < 1e-8, 1.0, rng)
    lo = w.bounds[0].copy()
    if w.task_col is not None:
        lo[w.task_col], inv_range[w.task_col] = 0.0, 1.0
    assert np.array_equal(a["xn"], (w.train_x - lo) * inv_range)
    K, dK = host_gram(a["xn"], w, row.outputscale or 1.0, m.jitter)
    absL = np.abs(L)
    chol_err = np.tril(np.abs(L @ L.T - K))
    chol = _ratio(chol_err, np.tril(gamma(n + 1) * (absL @ absL.T) + dK))
    inv = _ratio(np.abs(L @ X - np.eye(n)), inverse_bound(L, X))

    # b. derived arrays
    r = a["r"]
    aX = np.abs(X)
    alpha_ref = X.T @ (X @ r)
    alpha = _ratio(np.abs(a["alpha64"] - alpha_ref), gamma(n) * (aX.T @ (aX @ np.abs(r))))
    resid = _ratio(np.abs(K @ a["alpha64"] - r), n * U * (np.abs(K) @ np.abs(a["alpha64"]) + np.abs(r)))
    n_pad = m.n_pad
    assert np.array_equal(a["alpha32"][:n], a["alpha64"].astype(np.float32))
    assert not a["alpha32"][n:].any()
    Xp = np.zeros((n_pad, n_pad))
    Xp[:n, :n] = X
    assert np.array_equal(a["linv32"], Xp.astype(np.float32))
    s = float(m.r_scale)
    assert 2.0 ** 13 <= s * np.abs(X).max() < 2.0 ** 14
    v = s * Xp
    img = decode_rimg(a["rimg"], m.n_chunks)
    assert np.array_equal(img[v == 0.0], v[v == 0.0]), "tensor-core image: non-zero outside L^-1"
    rimg = _ratio(np.abs(img - v), 2.0 ** -22 * np.abs(v) + 2.0 ** -25)
    _report(row.name, chol=chol, inv=inv, alpha=alpha, resid=resid, rimg=rimg)
    assert chol <= 2.0 and inv <= 2.0 and alpha <= 4.0 and rimg <= 2.0 and resid <= 4.0
    # the float64 caches equal the oracle's to its forward error (a gross cross-check: wrong data, wrong scaling)
    assert np.abs(X - om.R.numpy().T).max() <= 1e-6 * np.abs(X).max()


# ------------------------------------------------------------------------------------------
# GPU: d. joint posterior and pending statistics
# ------------------------------------------------------------------------------------------
def _oracle_joint(om, gp, rows32: np.ndarray):
    """oracle.posterior_joint on the device's own inputs: fp32 rows normalised with the fp32 bounds, fp32 y
    statistics (test_gpu_nei.py) and the fp32 mean constant; returns (mu, cov, beta = K^-1 k(X, rows))."""
    from oracle.reference_path import _kernel_diag, _standardised_posterior, kernel_matrix

    f32 = lambda v: torch.as_tensor(np.asarray(v, dtype=np.float32), dtype=torch.float64)  # noqa: E731
    Xn = (f32(rows32) - f32(om.lo)) * f32(1.0 / om.rng.numpy())
    _, mean, V = _standardised_posterior(om, Xn)
    tid = oracle.reference_path._task_ids(Xn, om.spec.task_idx)
    mean = mean - om.mean_const[tid] + f32(om.mean_const.numpy())[tid]  # bb_model keeps the mean constant in fp32
    c = kernel_matrix(om.spec, Xn, Xn) - V @ V.T
    c.diagonal().copy_(_kernel_diag(om.spec, Xn) - (V * V).sum(-1))
    ys, ym = float(np.float32(om.y_std)), float(np.float32(om.y_mean))
    beta = (om.R @ V.T).T
    return (ym + ys * mean).numpy(), (ys * ys * c).numpy(), beta.numpy(), Xn


def joint_tolerances(om, Xn: torch.Tensor):
    """(mu, cov, beta) tolerance factors c u (n kappa + d + A2) times their scales (module docstring, d.)."""
    n, d = om.n, om.d
    ev = torch.linalg.eigvalsh(om.L @ om.L.T)
    kappa = float(ev[-1] / ev[0])
    ls = np.ones(d)
    ls[om.spec.active_dims] = om.spec.lengthscale
    act = np.zeros(d, dtype=bool)
    act[om.spec.active_dims] = True
    cen = om.Xn.numpy().mean(axis=0)
    A2 = max(float((((x.numpy()[:, act] - cen[act]) / ls[act]) ** 2).sum(axis=1).max()) for x in (Xn, om.Xn))
    kmax = float(om.spec.outputscale or 1.0) * (1.0 if om.spec.task_covar is None
                                                else float(np.diag(om.spec.task_covar).max()))
    f = 8 * U * (n * kappa + d + A2)
    ys = float(np.float32(om.y_std))
    return (f * ys * (1.0 + float(np.abs(om.alpha.numpy()).sum()) * kmax), f * ys * ys * kmax, f), kappa


def _joint_rows(w: Workload, R: int) -> np.ndarray:
    k = min(R // 2, len(w.train_x))
    return np.concatenate([w.train_x[:k], w.candidates[:R - k]]).astype(np.float32)


def check_joint(gp, om, w: Workload, Rs, Ps, name: str):
    from baybe_b200 import noisy

    for R in Rs:
        rows = _joint_rows(w, R)
        mu, cov, (px, beta) = noisy._joint_posterior(gp, rows, with_beta=True)
        beta = beta.cpu().numpy()
        rmu, rcov, rbeta, Xn = _oracle_joint(om, gp, rows)
        (tmu, tcov, fb), kappa = joint_tolerances(om, Xn)
        assert beta.shape == (R, gp.model.n_pad) and not beta[:, gp.model.n:].any()
        bt = EPS32 * np.abs(rbeta) + fb * np.abs(rbeta).max(axis=1, keepdims=True)
        ratios = dict(mu=float(np.abs(mu - rmu).max() / tmu), cov=float(np.abs(cov - rcov).max() / tcov),
                      beta=_ratio(np.abs(beta[:, :gp.model.n] - rbeta), bt))
        _report(f"{name} R={R} kappa={kappa:.2e}", **ratios)
        assert max(ratios.values()) <= 1.0
        assert np.array_equal(cov, cov.T)
        for P in Ps:
            if P > R:
                continue
            p, pbeta, pmu, pcov = gp.pending_stats(rows[:P])
            sub_mu, sub_cov, (_, sub_beta) = noisy._joint_posterior(gp, rows[:P], with_beta=True)
            # fp32 outputs are the float64 values rounded once
            assert torch.equal(pbeta, sub_beta) and torch.equal(pbeta, torch.from_numpy(beta[:P]).to(pbeta.device))
            assert np.array_equal(pmu.cpu().numpy(), sub_mu.astype(np.float32)), (pmu, sub_mu)
            assert np.array_equal(pcov.cpu().numpy(), sub_cov.astype(np.float32))
            assert np.array_equal(sub_mu, mu[:P]) and np.array_equal(sub_cov, cov[:P, :P])


JOINT_SHAPES = [r for r in SHAPES if r.joint]


@pytest.mark.gpu
@pytest.mark.parametrize("row", JOINT_SHAPES, ids=lambda r: r.name)
def test_joint_posterior_and_pending_stats_float64(row, cuda_device):
    from baybe_b200 import DeviceGP

    n_pad = layout(row.n, row.width())["n_pad"]
    w = workload(row, n_query=n_pad)
    gp = DeviceGP(device=cuda_device, **w.gp_kwargs())
    assert gp.model.n_pad == n_pad
    check_joint(gp, oracle_model(w), w, sorted({1, 31, 32, n_pad}), (1, 31), row.name)


@pytest.mark.gpu
def test_pending_stats_of_a_4096_bit_fingerprint_model(cuda_device):
    """d + 2n = 6144 > 5888: 51 200 bytes of shared memory for k_pending_w, above the default 48 KB launch limit."""
    from baybe_b200 import DeviceGP

    w = fingerprint_workload(N=1200, d=4096, n=1024, seed=3)
    w.candidates = np.delete(w.candidates, w.train_idx, axis=0)
    gp = DeviceGP(device=cuda_device, **w.gp_kwargs())
    assert gp.model.wide and gp.model.n == 1024 and gp.model.d == 4096
    check_joint(gp, oracle_model(w), w, (31, 64), (31,), "fingerprint4096_n1024")


# ------------------------------------------------------------------------------------------
# GPU: e. fit objective
# ------------------------------------------------------------------------------------------
FIT_D = 4


def fit_problem(n: int, T: int, seed: int):
    rng = np.random.default_rng(seed)
    X = rng.random((n, FIT_D))
    tid = None if T == 1 else (np.arange(n) % T).astype(np.int32)
    y = smooth_target(X) + 0.01 * rng.standard_normal(n)
    y = (y - y.mean()) / y.std(ddof=1)
    W = rng.uniform(0.2, 1.0, (T, T))
    B = W @ W.T + np.diag(rng.uniform(0.1, 0.5, T))
    B /= B.max()
    theta = np.concatenate([rng.uniform(0.3, 1.5, FIT_D), [rng.uniform(1e-3, 2e-2)], [rng.normal(0, 0.3)],
                            B.reshape(-1)])
    return X, y, tid, B, theta


def fit_condition(X, tid, B, theta, family) -> float:
    """cond(K) of the fit's Gram matrix, from the oracle's kernel."""
    n, d = X.shape
    T = B.shape[0]
    Xt = torch.as_tensor(np.concatenate([X, (np.zeros(n) if tid is None else tid)[:, None]], axis=1))
    spec = oracle.KernelSpec(family=family, lengthscale=theta[:d], active_dims=list(range(d)),
                             task_idx=d, task_covar=B.reshape(T, T))
    K = oracle.kernel_matrix(spec, Xt, Xt)
    K.diagonal().copy_(torch.as_tensor(np.diag(B)[np.zeros(n, dtype=int) if tid is None else tid]))
    K = K + float(theta[d]) * torch.eye(n, dtype=torch.float64)
    ev = torch.linalg.eigvalsh(K)
    return float(ev[-1] / ev[0])


@pytest.mark.gpu
@pytest.mark.parametrize("criterion", ["mll", "loo"])
@pytest.mark.parametrize("T", [1, 4, 16])
@pytest.mark.parametrize("n", [33, 129, 513, 1024])
def test_fit_objective_at_block_boundaries(n, T, criterion, cuda_device):
    from baybe_b200.surrogates import DeviceMLL

    family = (M52, RBF, M32, M12)[(n + T) % 4]
    X, y, tid, B, theta = fit_problem(n, T, seed=7 * n + T)
    dev = DeviceMLL(X, y, tid, T, family, cuda_device, criterion=criterion)
    host = HostMLL(X, y, tid, T, family, criterion=criterion)
    val, grad, ok = dev(theta)
    rval, rgrad, rok = host(theta)
    assert ok and rok, "not_pd must be 0"
    kappa = fit_condition(X, tid, B, theta, family)
    f = n * U * kappa
    rv = abs(val - rval) / (f * max(1.0, abs(rval)))
    rg = float(np.abs(grad - rgrad).max()) / (f * max(1.0, float(np.abs(rgrad).max())))
    _report(f"fit {criterion} n={n} T={T} {family} kappa={kappa:.2e}", value=rv, grad=rg)
    assert rv <= 1.0 and rg <= 1.0


# ------------------------------------------------------------------------------------------
# GPU: f. jitter escalation
# ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("delta", list(JITTER_CASES))
def test_jitter_escalation_matches_psd_safe_cholesky(delta, cuda_device):
    from baybe_b200 import DeviceGP
    from baybe_b200.surrogates import DeviceMLL

    kw = jitter_model(delta)
    want = JITTER_CASES[delta]
    n = len(kw["train_y"])
    if want is None:
        with pytest.raises(FloatingPointError, match="not positive definite"):
            DeviceGP(device=cuda_device, **kw)
    else:
        gp = DeviceGP(device=cuda_device, **kw)
        om = _oracle_jitter_model(kw)
        assert (gp.model.jitter_tries, gp.model.jitter) == want and gp.model.jitter == om.jitter
        # the factor of K + jitter I, and its inverse, within the bounds of test_model_build_float64
        a = device_arrays(gp)
        K = kw["task_covar"][kw["train_x"][:, 1].astype(int)][:, kw["train_x"][:, 1].astype(int)]
        K = K + (1e-4 + gp.model.jitter) * np.eye(n)
        L, X = a["L"], a["X"]
        chol = _ratio(np.tril(np.abs(L @ L.T - K)), np.tril(gamma(n + 1) * (np.abs(L) @ np.abs(L).T)))
        inv = _ratio(np.abs(L @ X - np.eye(n)), inverse_bound(L, X))
        _report(f"jitter delta={delta:g}", chol=chol, inv=inv)
        assert chol <= 2.0 and inv <= 2.0
    # the fit objective has no jitter: the same K (kernel 1 between identical rows, B, noise 1e-4) is not positive
    # definite there unless its smallest eigenvalue already is positive
    tid = kw["train_x"][:, 1].astype(np.int32)
    mll = DeviceMLL(kw["train_x"][:, :1], np.zeros(n), tid, 2, RBF, cuda_device)
    _, _, ok = mll(np.concatenate([[0.7], [1e-4], [0.0], kw["task_covar"].reshape(-1)]))
    assert ok == (delta < 0)
