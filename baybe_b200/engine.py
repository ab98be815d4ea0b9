"""Host side of the scoring engine: PyTorch owns device memory and streams, every numeric step
is a C-ABI call into ``libbaybe_b200.so`` (hand-written sm_90a CUDA).  The calls are exposed
as ``torch.library`` custom ops in the ``baybe_b200::`` namespace so that they compose with
``torch.no_grad`` code the way the reference's BoTorch calls do.

Replaces the L1 layer of SURVEY.md section 1: ``model.posterior`` / ``acqf.forward`` /
``optimize_acqf_discrete`` as reached from
``/root/reference/baybe/recommenders/pure/bayesian/botorch/discrete.py:120-126``.
"""

from __future__ import annotations

import ctypes as C
import os
import itertools
import math
import threading
import weakref
from dataclasses import dataclass

import numpy as np
import torch

from baybe_b200 import _lib

__all__ = ["AcqConfig", "DeviceGP", "sobol_normal_samples", "pack_best", "unpack_best", "decode_best", "DEFAULT_MC_SAMPLES"]

DEFAULT_MC_SAMPLES = 512  # botorch MC acquisition default sample shape
# handle -> model; weak, so a model dropped without close() (a new recommender per BO iteration) frees its device
# blob with the last strong reference instead of living as long as the process
_registry: "weakref.WeakValueDictionary[int, DeviceGP]" = weakref.WeakValueDictionary()
_registry_lock = threading.Lock()
_handle_counter = itertools.count(1)


def _stream_ptr() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t: torch.Tensor | None) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


def _require_cuda(device: torch.device | str | None) -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError(
            "baybe_b200 needs a CUDA device (sm_90a); there is no CPU fallback for the scoring path"
        )
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(f"baybe_b200 runs on CUDA devices only, got {dev}")
    return dev


def sobol_normal_samples(n_samples: int, dim: int, seed: int) -> torch.Tensor:
    """Base samples exactly as botorch's ``SobolQMCNormalSampler`` draws them (SURVEY A.6):
    scrambled Sobol -> v = 0.5 + (1-eps)(u-0.5) -> sqrt(2) erfinv(2v-1); float64 (S, dim) on CPU.
    The engine takes base samples as an explicit input so that any checker shares them."""
    eng = torch.quasirandom.SobolEngine(dimension=dim, scramble=True, seed=seed)
    u = eng.draw(n_samples, dtype=torch.float64)
    v = 0.5 + (1.0 - torch.finfo(torch.float64).eps) * (u - 0.5)
    return torch.erfinv(2.0 * v - 1.0) * math.sqrt(2.0)


@dataclass(frozen=True)
class AcqConfig:
    """Acquisition kind + context, the content of ``bb_acq_spec`` (include/baybe_b200.h)."""

    kind: str
    best_f: float = 0.0
    beta: float = 0.2
    obj_scale: float = 1.0
    obj_shift: float = 0.0
    maximize: bool = True
    tau_relu: float = 1e-6
    tau_max: float = 1e-2
    tau_pi: float = 1e-3

    def __post_init__(self):
        if self.kind not in (tuple(_lib.ACQ_KIND) + _lib.NEI_KINDS + _lib.PAREGO_KINDS + _lib.NEHVI_KINDS
                             + _lib.NIPV_KINDS):
            raise ValueError(f"unsupported acquisition function {self.kind!r}")

    @property
    def is_mc(self) -> bool:
        return self.kind in _lib.MC_KINDS + _lib.NEI_KINDS + _lib.PAREGO_KINDS + _lib.NEHVI_KINDS + _lib.NIPV_KINDS

    def to_c(self) -> _lib.AcqSpec:
        if self.kind in _lib.NEI_KINDS:
            raise NotImplementedError(f"{self.kind} is evaluated by baybe_b200.noisy.NeiScorer (discrete spaces) or "
                                      "baybe_b200.hybrid.NeiScorer (hybrid spaces), not by the fused kernels")
        if self.kind in _lib.PAREGO_KINDS:
            raise NotImplementedError(f"{self.kind} is evaluated by baybe_b200.parego.ParegoScorer, not by the fused "
                                      "kernels")
        if self.kind in _lib.NEHVI_KINDS:
            raise NotImplementedError(f"{self.kind} is evaluated by baybe_b200.nehvi.NehviScorer, not by the fused "
                                      "kernels")
        if self.kind in _lib.NIPV_KINDS:
            raise NotImplementedError(f"{self.kind} is evaluated by baybe_b200.nipv.NipvScorer, not by the fused "
                                      "kernels")
        return _lib.AcqSpec(
            _lib.ACQ_KIND[self.kind], int(self.maximize), self.best_f, self.beta, self.obj_scale,
            self.obj_shift, self.tau_relu, self.tau_max, self.tau_pi,
        )

    def params(self) -> list[float]:
        return [float(self.maximize), self.best_f, self.beta, self.obj_scale, self.obj_shift,
                self.tau_relu, self.tau_max, self.tau_pi]

    @staticmethod
    def from_params(kind_id: int, prm: list[float]) -> "AcqConfig":
        kind = {v: k for k, v in _lib.ACQ_KIND.items()}[kind_id]
        return AcqConfig(kind, prm[1], prm[2], prm[3], prm[4], bool(prm[0]), prm[5], prm[6], prm[7])


def _layout_of(x: torch.Tensor) -> tuple[int, int]:
    """(bb_layout code, leading dimension) of a 2-D device tensor; no copy if it is row-major or
    column-major (the reference hands BoTorch a float64 column-major matrix,
    baybe/utils/dataframe.py:68-81)."""
    n, d = x.shape
    if x.dtype == torch.uint8:  # bit-packed binary features: rows of bytes
        if n > 1 and x.stride(1) != 1:
            raise ValueError("bit-packed candidate rows must be contiguous")
        return (_lib.LAYOUT["bits_u8"], int(x.stride(0)) if n > 1 else d)
    if x.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"candidate dtype must be float32, float64 or uint8 (bit-packed), got {x.dtype}")
    f64 = x.dtype == torch.float64
    s0, s1 = x.stride()
    # a single row / single column carries no layout of its own: it is whatever its strides say.  The
    # column-major test comes FIRST so that a one-row slice of a column-major matrix (strides (1, N), what the
    # reference hands over) is read with ld = N, and nothing here ever copies: the caller passes x.data_ptr().
    if s0 == 1 and s1 >= n and not (s1 == 1 and s0 >= d):
        return (_lib.LAYOUT["col_f64" if f64 else "col_f32"], int(s1))
    if s1 == 1 and (s0 >= d or n <= 1):
        return (_lib.LAYOUT["row_f64" if f64 else "row_f32"], max(int(s0), d) if n > 1 else d)
    if d <= 1 and s0 >= 1:  # one column, rows s0 apart: row-major with ld = s0
        return (_lib.LAYOUT["row_f64" if f64 else "row_f32"], int(s0))
    raise ValueError("candidate matrix must be row-major or column-major (call .contiguous())")


def _as_device_matrix(x, device: torch.device, d: int) -> torch.Tensor:
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(x)
    if x.dim() == 2 and x.dtype == torch.uint8:  # bit-packed rows (BB_BITS_U8)
        if x.shape[1] != (d + 7) // 8:
            raise ValueError(f"expected a bit-packed (N, {(d + 7) // 8}) uint8 matrix, got {tuple(x.shape)}")
        return x.to(device, non_blocking=True).contiguous()
    if x.dim() != 2 or x.shape[1] != d:
        raise ValueError(f"expected a (N, {d}) candidate matrix, got {tuple(x.shape)}")
    if x.dtype not in (torch.float32, torch.float64):
        x = x.to(torch.float64)
    if x.device != device:
        x = x.to(device, non_blocking=True)
    s0, s1 = x.stride()
    n = x.shape[0]
    ok_row = s1 == 1 and (s0 >= d or n <= 1)
    ok_col = s0 == 1 and s1 >= n
    if not (ok_row or ok_col):  # anything else (e.g. x[:1, ::2]) is copied HERE, where the caller sees it
        x = x.contiguous()
    return x


class DeviceGP:
    """Device-resident fitted GP: the caches gpytorch builds on the first posterior call
    (Cholesky root, alpha, inverse root) plus their tensor-core image, built by
    ``bb_model_build`` from fixed hyper-parameters.

    Args mirror what ``GaussianProcessSurrogate._fit`` passes to ``botorch.models.SingleTaskGP``
    (``/root/reference/baybe/surrogates/gaussian_process/core.py:301-339``) after fitting:
      train_x (n,d) raw comp-rep, train_y (n,), bounds (2,d) = searchspace.scaling_bounds,
      family in {matern12, matern32, matern52, rbf}, lengthscale (d,) with <=0 for inactive
      columns, noise / mean_const scalars or (T,), outputscale or None, task_col or None,
      task_covar (T,T) or None.
    """

    def __init__(self, train_x, train_y, bounds, family: str, lengthscale, noise, mean_const=0.0,
                 outputscale: float | None = None, task_col: int | None = None, task_covar=None,
                 device: torch.device | str | None = None):
        self.device = _require_cuda(device)
        lib = _lib.load()
        tx = np.ascontiguousarray(np.asarray(train_x, dtype=np.float64))
        ty = np.ascontiguousarray(np.asarray(train_y, dtype=np.float64).reshape(-1))
        if tx.ndim != 2 or tx.shape[0] != ty.shape[0]:
            raise ValueError("train_x must be (n,d) and train_y (n,)")
        n, d = tx.shape
        bnd = np.ascontiguousarray(np.asarray(bounds, dtype=np.float64))
        if bnd.shape != (2, d):
            raise ValueError(f"bounds must be (2,{d})")
        if family not in _lib.KERNEL_FAMILY:
            raise ValueError(f"unknown kernel family {family!r}")
        T = 1 if task_covar is None else int(np.asarray(task_covar).shape[0])
        if (task_col is None) != (task_covar is None):
            raise ValueError("task_col and task_covar must be given together")
        ls = np.ascontiguousarray(np.broadcast_to(np.asarray(lengthscale, dtype=np.float64), (d,)))
        nz = np.ascontiguousarray(np.broadcast_to(np.asarray(noise, dtype=np.float64), (T,)))
        mc = np.ascontiguousarray(np.broadcast_to(np.asarray(mean_const, dtype=np.float64), (T,)))
        tcv = None if task_covar is None else np.ascontiguousarray(np.asarray(task_covar, dtype=np.float64))
        self.n, self.d, self.n_tasks = n, d, T
        self.family, self.task_col = family, task_col
        self.outputscale = None if outputscale is None else float(outputscale)
        # the fitted hyper-parameters as given: lengthscale (d,), likelihood noise per task (T,), task covariance
        # (T, T) or None
        self.lengthscale, self.noise, self.task_covar = ls, nz, tcv
        self._keepalive = (tx, ty, bnd, ls, nz, mc, tcv)
        dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
        lo_arr, hi_arr = np.ascontiguousarray(bnd[0]), np.ascontiguousarray(bnd[1])
        desc = _lib.ModelDesc(
            n, d, _lib.KERNEL_FAMILY[family], -1 if task_col is None else int(task_col), T,
            int(outputscale is not None), float(outputscale or 1.0),
            dp(tx), dp(ty), dp(lo_arr), dp(hi_arr), dp(ls), dp(nz), dp(mc),
            None if tcv is None else dp(tcv),
        )
        nbytes = lib.bb_model_blob_bytes(n, d, T)
        if nbytes == 0:
            raise ValueError("invalid model dimensions")
        with torch.cuda.device(self.device):
            # 1024-byte aligned caller-owned blob
            self._blob = torch.empty(nbytes + 1024, dtype=torch.uint8, device=self.device)
            base = (self._blob.data_ptr() + 1023) // 1024 * 1024
            self.model = _lib.Model()
            _lib.check(lib.bb_model_build(C.byref(desc), C.c_void_p(base), nbytes,
                                          C.byref(self.model), _stream_ptr()), "bb_model_build")
        self.train_x = tx
        self.handle = next(_handle_counter)
        with _registry_lock:
            _registry[self.handle] = self

    def close(self) -> None:
        with _registry_lock:
            _registry.pop(self.handle, None)

    # ---- tensors -----------------------------------------------------------------------
    def prepare(self, x) -> torch.Tensor:
        """Move a candidate matrix to this model's device (no-op if already there)."""
        return _as_device_matrix(x, self.device, self.d)

    # ---- hot-path calls (all via torch custom ops -> C ABI) -----------------------------
    def kernel_matrix(self, x) -> torch.Tensor:
        return torch.ops.baybe_b200.kernel_matrix(self.prepare(x), self.handle)

    def posterior(self, x) -> tuple[torch.Tensor, torch.Tensor]:
        """Marginal posterior mean / variance (float32, original units) of every row of x."""
        return torch.ops.baybe_b200.posterior(self.prepare(x), self.handle)

    def posterior_simt(self, x) -> tuple[torch.Tensor, torch.Tensor]:
        """Test-only diagnostic path (plain fp32 SIMT, no tensor cores)."""
        return torch.ops.baybe_b200.posterior_simt(self.prepare(x), self.handle)

    def pending_stats(self, pending) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """(pending fp32 rows, beta [P,n_pad], mean [P], covariance [P,P]) of pending points."""
        p = torch.as_tensor(np.asarray(pending, dtype=np.float32) if not torch.is_tensor(pending) else pending)
        p = p.to(self.device, torch.float32).reshape(-1, self.d).contiguous()
        beta, mu, cov = torch.ops.baybe_b200.pending_stats(p, self.handle)
        return p, beta, mu, cov

    def cross_covariance(self, x, pend_x: torch.Tensor, beta: torch.Tensor):
        return torch.ops.baybe_b200.posterior_cross(self.prepare(x), pend_x, beta, self.handle)

    def score(self, acq: AcqConfig, x, z: torch.Tensor | None, keep: torch.Tensor | None = None,
              index_offset: int = 0, want_scores: bool = True):
        """One fused pass: posterior + q=1 acquisition + arg-max.  Returns (scores or None,
        packed best key (int64 device tensor of shape [1])).

        A large candidate matrix living in (ideally pinned) HOST memory is streamed: row blocks are
        copied on a side stream while the previous block is being scored, so the pass costs about
        max(H2D, compute) instead of their sum."""
        zf = None
        if acq.is_mc:
            if z is None:
                raise ValueError("Monte Carlo acquisition functions need base samples")
            zf = z.reshape(-1).to(self.device, torch.float32)
        if torch.is_tensor(x) and x.device.type == "cpu" and x.dim() == 2 and x.shape[0] >= self.STREAM_MIN_ROWS \
                and x.dtype in (torch.float32, torch.float64) and x.is_contiguous():
            return self._score_streamed(acq, x, zf, keep, index_offset, want_scores)
        xd = self.prepare(x)
        return torch.ops.baybe_b200.score_fused(xd, keep, zf, self.handle, _lib.ACQ_KIND[acq.kind],
                                                acq.params(), int(index_offset), bool(want_scores))

    STREAM_MIN_ROWS = 262_144
    STREAM_BLOCKS = 8
    # single-launch gated pass where the headline kernel covers the shape.  BB_OVERLAPPED_HOST_PASS=0 selects the
    # block-wise pass: needed under ncu, whose kernel serialisation keeps the copy stream from making progress while
    # the gated kernel waits for it (every such launch then runs into its 2 s time-out)
    OVERLAPPED_HOST_PASS = os.environ.get("BB_OVERLAPPED_HOST_PASS", "1") != "0"

    def _host_pass(self, acq: AcqConfig, h: torch.Tensor, fmt: str, ld: int, row_bytes: int, table, zf, keep,
                   index_offset: int, want_scores: bool):
        """One ``bb_score_fused_host`` call: H2D of row blocks on the side stream overlapped with decode + scoring."""
        lib = _lib.load()
        N = h.shape[0]
        if self.OVERLAPPED_HOST_PASS and fmt != "rows_f64" and N > 0 and not self.model.wide:
            out = self._host_pass_overlapped(lib, acq, h, fmt, ld, row_bytes, table, zf, keep, index_offset, want_scores)
            if out is not None:
                return out
        rows = -(-N // self.STREAM_BLOCKS)
        rows = max(-(-rows // 128) * 128, 128)
        coded = fmt.startswith("codes")
        with torch.cuda.device(self.device):
            main = torch.cuda.current_stream()
            if not hasattr(self, "_copy_stream"):
                self._copy_stream = torch.cuda.Stream(device=self.device)
            key_ = (rows * row_bytes, rows if coded else 0)
            if getattr(self, "_stage_key", None) != key_:  # staging buffers are reused across calls
                self._stage = [torch.empty(rows * row_bytes, dtype=torch.uint8, device=self.device) for _ in range(2)]
                self._rowbuf = ([torch.empty((rows, self.d), dtype=torch.float32, device=self.device) for _ in range(2)]
                                if coded else [None, None])
                self._stage_key = key_
            score = torch.empty(N if want_scores else 0, dtype=torch.float32, device=self.device)
            key = torch.empty(1, dtype=torch.int64, device=self.device)
            c_acq = acq.to_c()
            stage = (C.c_void_p * 2)(self._stage[0].data_ptr(), self._stage[1].data_ptr())
            rowb = (C.c_void_p * 2)(*(0 if t is None else t.data_ptr() for t in self._rowbuf))
            S = 0 if zf is None else zf.numel()
            _lib.check(lib.bb_score_fused_host(
                C.byref(self.model), C.byref(c_acq), C.c_void_p(h.data_ptr()), _lib.HOST_FORMAT[fmt], N, ld,
                _ptr(table), 0 if table is None else table.shape[1], stage, rowb, rows, _ptr(keep), _ptr(zf), S,
                _ptr(score) if want_scores else None, _ptr(key), int(index_offset), _stream_ptr(),
                C.c_void_p(self._copy_stream.cuda_stream)), "bb_score_fused_host")
            self._copy_stream.wait_stream(main)  # later work on the side stream stays ordered behind this pass
        return score, key

    def _host_pass_overlapped(self, lib, acq, h, fmt, ld, row_bytes, table, zf, keep, index_offset, want_scores):
        """``bb_score_fused_overlapped``: one kernel launch that consumes the rows while the copy stream delivers
        them.  Returns None when the shape is outside the headline kernel's envelope (caller falls back)."""
        N = h.shape[0]
        with torch.cuda.device(self.device):
            main = torch.cuda.current_stream()
            if not hasattr(self, "_copy_stream"):
                self._copy_stream = torch.cuda.Stream(device=self.device)
            need = N * row_bytes
            if getattr(self, "_stage_all", None) is None or self._stage_all.numel() < need:
                self._stage_all = torch.empty(need, dtype=torch.uint8, device=self.device)
                self._gate = torch.zeros(2, dtype=torch.int32, device=self.device)  # [rows landed, status]
            score = torch.empty(N if want_scores else 0, dtype=torch.float32, device=self.device)
            key = torch.empty(1, dtype=torch.int64, device=self.device)
            c_acq = acq.to_c()
            S = 0 if zf is None else zf.numel()
            rc = lib.bb_score_fused_overlapped(
                C.byref(self.model), C.byref(c_acq), C.c_void_p(h.data_ptr()), _lib.HOST_FORMAT[fmt], N, ld,
                _ptr(table), 0 if table is None else table.shape[1], _ptr(self._stage_all), self._stage_all.numel(),
                C.c_void_p(self._gate.data_ptr()), C.c_void_p(self._gate.data_ptr() + 4), _ptr(keep), _ptr(zf), S,
                _ptr(score) if want_scores else None, _ptr(key), int(index_offset), _stream_ptr(),
                C.c_void_p(self._copy_stream.cuda_stream))
            if rc == _lib.BB_ERR_UNSUPPORTED:
                return None
            _lib.check(rc, "bb_score_fused_overlapped")
            self._copy_stream.wait_stream(main)
            self._gated_pass_pending = True
        return score, key

    def check_host_pass(self) -> None:
        """Raise if the last overlapped host pass saw rows that were never published (synchronises)."""
        if getattr(self, "_gated_pass_pending", False):
            self._gated_pass_pending = False
            if int(self._gate[1].item()) != 0:
                raise RuntimeError("bb_score_fused_overlapped: host rows were not published within the time-out")

    def _score_streamed(self, acq: AcqConfig, x: torch.Tensor, zf, keep, index_offset: int, want_scores: bool):
        if x.shape[1] != self.d:
            raise ValueError(f"expected a (N, {self.d}) candidate matrix, got {tuple(x.shape)}")
        f64 = x.dtype == torch.float64
        return self._host_pass(acq, x, "rows_f64" if f64 else "rows_f32", self.d, self.d * (8 if f64 else 4), None, zf,
                               keep, index_offset, want_scores)

    def score_coded(self, acq: AcqConfig, codes: torch.Tensor, table, bits: int, z: torch.Tensor | None,
                    keep: torch.Tensor | None = None, index_offset: int = 0, want_scores: bool = True):
        """``score`` for a LEVEL-CODED candidate matrix (``baybe_b200.bits.encode_levels``): rows of 4- or 8-bit
        level indices plus the per-column value table -- the compact, exact form of a discrete search space
        (d/2 or d bytes per candidate instead of 4d).  `codes` may live in (pinned) host memory: row blocks are
        copied on a side stream, expanded on the device by ``bb_decode_codes`` and scored, so the end-to-end pass
        moves 8x / 4x fewer bytes over PCIe than the float32 matrix.  Scores are bit-identical to ``score`` on the
        decoded float32 matrix."""
        if bits not in (4, 8):
            raise ValueError("bits must be 4 or 8")
        if codes.dtype != torch.uint8 or codes.dim() != 2 or not codes.is_contiguous():
            raise ValueError("codes must be a contiguous 2-D uint8 tensor")
        row_bytes = (self.d + 1) // 2 if bits == 4 else self.d
        if codes.shape[1] != row_bytes:
            raise ValueError(f"expected {row_bytes} code bytes per row, got {codes.shape[1]}")
        tab = torch.as_tensor(np.asarray(table, dtype=np.float32) if not torch.is_tensor(table) else table)
        tab = tab.to(self.device, torch.float32).contiguous()
        if tab.dim() != 2 or tab.shape[0] != self.d or tab.shape[1] > (1 << bits):
            raise ValueError(f"value table must be ({self.d}, <= {1 << bits})")
        zf = None
        if acq.is_mc:
            if z is None:
                raise ValueError("Monte Carlo acquisition functions need base samples")
            zf = z.reshape(-1).to(self.device, torch.float32)
        if codes.device.type == "cpu":
            return self._host_pass(acq, codes, "codes4" if bits == 4 else "codes8", row_bytes, row_bytes, tab, zf, keep,
                                   index_offset, want_scores)
        lib = _lib.load()
        N = codes.shape[0]
        with torch.cuda.device(self.device):  # device-resident codes: expand once, score
            rows = torch.empty((N, self.d), dtype=torch.float32, device=self.device)
            _lib.check(lib.bb_decode_codes(_ptr(codes), bits, N, self.d, row_bytes, _ptr(tab), tab.shape[1], _ptr(rows),
                                           self.d, _stream_ptr()), "bb_decode_codes")
        return torch.ops.baybe_b200.score_fused(rows, keep, zf, self.handle, _lib.ACQ_KIND[acq.kind], acq.params(),
                                                int(index_offset), bool(want_scores))

    def score_joint(self, acq: AcqConfig, x, pending, z: torch.Tensor) -> torch.Tensor:
        """MC acquisition value of [x*; pending] for every row x* (sequential-greedy round)."""
        xd = self.prepare(x)
        px, beta, pmu, pcov = self.pending_stats(pending)
        mu, var, cross = self.cross_covariance(xd, px, beta)
        zf = z.to(self.device, torch.float32).contiguous()
        return torch.ops.baybe_b200.acq_score_joint(mu, var, cross, pmu, pcov, zf,
                                                    _lib.ACQ_KIND[acq.kind], acq.params())

    def value_and_grad(self, acq: AcqConfig, x, z: torch.Tensor | None, pending=None):
        """Acquisition value [N] and its gradient [N, d] with respect to the raw comp-rep rows x (``bb_acq_grad``, or
        ``bb_acq_grad_large`` for wide models and n_pad > 256: ``acq_grad_op``).  Without pending points the value is
        ``score``'s; with them (Monte Carlo kinds, z of shape (S, 1 + p)) it is ``score_joint``'s value of
        [x; pending], candidate first."""
        xd = self.prepare(x).to(torch.float32).contiguous()
        zf = None
        if acq.is_mc:
            if z is None:
                raise ValueError("Monte Carlo acquisition functions need base samples")
            zf = z.to(self.device, torch.float32).contiguous()
        op = acq_grad_op(self.model)
        if pending is None or len(pending) == 0:
            return op(xd, None, None, None, None, zf, self.handle, _lib.ACQ_KIND[acq.kind], acq.params())
        px, beta, pmu, pcov = self.pending_stats(pending)
        return op(xd, px, beta, pmu, pcov, zf, self.handle, _lib.ACQ_KIND[acq.kind], acq.params())

    def argmax(self, scores: torch.Tensor, keep: torch.Tensor | None, index_offset: int = 0) -> torch.Tensor:
        """Packed (score, lowest global index) key of a score vector (``bb_argmax``)."""
        return torch.ops.baybe_b200.argmax(scores, keep, int(index_offset))

    def best_f(self, acq: AcqConfig) -> float:
        """max_i o(mu(x_i)) over the training inputs (baybe/acquisition/_builder.py:256-265)."""
        mu, _ = self.posterior(torch.from_numpy(self.train_x))
        return float((acq.obj_scale * mu.double() + acq.obj_shift).max().item())


def decode_best(key: torch.Tensor) -> tuple[float, int]:
    """(value, global index) of a packed best key; index -1 if nothing was eligible."""
    out = torch.ops.baybe_b200.best_decode(key)
    val = float(out[0].item())
    idx = int(out[1].item())
    return val, idx


def pack_best(score: float, idx: int) -> int:
    """Host-side twin of ``pack_key`` (csrc/common.cuh): signed-int64 order == (score, then lowest
    index; -0.0 packs as +0.0, so the zeros tie as in torch.argmax).  Used by the CPU tests of the sharded
    arg-max protocol."""
    import struct

    u = struct.unpack("<i", struct.pack("<f", score))[0]
    if u == -(1 << 31):  # -0.0
        u = 0
    s = u ^ ((u >> 31) & 0x7FFFFFFF)
    v = ((s & 0xFFFFFFFF) << 32) | (0xFFFFFFFF - idx)
    return v - (1 << 64) if v >= (1 << 63) else v


def unpack_best(key: int) -> tuple[float, int]:
    """Host-side decode of a packed (score, lowest index) key -- same bit layout as
    ``pack_key`` in csrc/common.cuh; (-inf, -1) for the empty key."""
    import struct

    if key == -(1 << 63):
        return float("-inf"), -1
    hi = (key >> 32) & 0xFFFFFFFF
    s = hi - (1 << 32) if hi & 0x80000000 else hi
    s ^= (s >> 31) & 0x7FFFFFFF
    val = struct.unpack("<f", struct.pack("<i", s))[0]
    return val, 0xFFFFFFFF - (key & 0xFFFFFFFF)


# ------------------------------------------------------------------------------------------
# torch.library custom ops (thin: allocate outputs with torch, call the C ABI on the current stream)
# ------------------------------------------------------------------------------------------
def _gp(handle: int) -> DeviceGP:
    try:
        return _registry[handle]
    except KeyError:
        raise RuntimeError(f"unknown baybe_b200 model handle {handle}") from None


@torch.library.custom_op("baybe_b200::kernel_matrix", mutates_args=())
def _op_kernel_matrix(x: torch.Tensor, handle: int) -> torch.Tensor:
    gp = _gp(handle)
    lay, ld = _layout_of(x)
    N = x.shape[0]
    out = torch.empty((N, gp.n), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().bb_kernel_matrix(C.byref(gp.model), _ptr(x), lay, N, ld, _ptr(out), gp.n,
                                                _stream_ptr()), "bb_kernel_matrix")
    return out


@_op_kernel_matrix.register_fake
def _(x, handle):
    return x.new_empty((x.shape[0], _gp(handle).n), dtype=torch.float32)


@torch.library.custom_op("baybe_b200::posterior", mutates_args=())
def _op_posterior(x: torch.Tensor, handle: int) -> tuple[torch.Tensor, torch.Tensor]:
    gp = _gp(handle)
    lay, ld = _layout_of(x)
    N = x.shape[0]
    mu = torch.empty(N, dtype=torch.float32, device=x.device)
    var = torch.empty(N, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().bb_posterior(C.byref(gp.model), _ptr(x), lay, N, ld, _ptr(mu), _ptr(var),
                                            None, None, None, 0, _stream_ptr()), "bb_posterior")
    return mu, var


@_op_posterior.register_fake
def _(x, handle):
    return x.new_empty(x.shape[0], dtype=torch.float32), x.new_empty(x.shape[0], dtype=torch.float32)


@torch.library.custom_op("baybe_b200::posterior_simt", mutates_args=())
def _op_posterior_simt(x: torch.Tensor, handle: int) -> tuple[torch.Tensor, torch.Tensor]:
    gp = _gp(handle)
    lay, ld = _layout_of(x)
    N = x.shape[0]
    mu = torch.empty(N, dtype=torch.float32, device=x.device)
    var = torch.empty(N, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().bb_debug_posterior_simt(C.byref(gp.model), _ptr(x), lay, N, ld, _ptr(mu),
                                                       _ptr(var), _stream_ptr()), "bb_debug_posterior_simt")
    return mu, var


@_op_posterior_simt.register_fake
def _(x, handle):
    return x.new_empty(x.shape[0], dtype=torch.float32), x.new_empty(x.shape[0], dtype=torch.float32)


@torch.library.custom_op("baybe_b200::pending_stats", mutates_args=())
def _op_pending_stats(pend_x: torch.Tensor, handle: int) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    gp = _gp(handle)
    P = pend_x.shape[0]
    beta = torch.empty((P, gp.model.n_pad), dtype=torch.float32, device=pend_x.device)
    mu = torch.empty(P, dtype=torch.float32, device=pend_x.device)
    cov = torch.empty((P, P), dtype=torch.float32, device=pend_x.device)
    with torch.cuda.device(pend_x.device):
        _lib.check(_lib.load().bb_pending_stats(C.byref(gp.model), _ptr(pend_x), P, _ptr(beta), _ptr(mu),
                                                _ptr(cov), _stream_ptr()), "bb_pending_stats")
    return beta, mu, cov


@_op_pending_stats.register_fake
def _(pend_x, handle):
    P = pend_x.shape[0]
    return (pend_x.new_empty((P, _gp(handle).model.n_pad)), pend_x.new_empty(P), pend_x.new_empty((P, P)))


@torch.library.custom_op("baybe_b200::posterior_cross", mutates_args=())
def _op_posterior_cross(x: torch.Tensor, pend_x: torch.Tensor, beta: torch.Tensor,
                        handle: int) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    gp = _gp(handle)
    lay, ld = _layout_of(x)
    N, P = x.shape[0], pend_x.shape[0]
    mu = torch.empty(N, dtype=torch.float32, device=x.device)
    var = torch.empty(N, dtype=torch.float32, device=x.device)
    cross = torch.empty((N, P), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().bb_posterior(C.byref(gp.model), _ptr(x), lay, N, ld, _ptr(mu), _ptr(var),
                                            _ptr(cross), _ptr(pend_x), _ptr(beta), P, _stream_ptr()),
                   "bb_posterior")
    return mu, var, cross


@_op_posterior_cross.register_fake
def _(x, pend_x, beta, handle):
    N, P = x.shape[0], pend_x.shape[0]
    f = dict(dtype=torch.float32)
    return x.new_empty(N, **f), x.new_empty(N, **f), x.new_empty((N, P), **f)


@torch.library.custom_op("baybe_b200::acq_score", mutates_args=())
def _op_acq_score(mu: torch.Tensor, var: torch.Tensor, z: torch.Tensor | None, kind: int,
                  params: list[float]) -> torch.Tensor:
    acq = AcqConfig.from_params(kind, params).to_c()
    N = mu.shape[0]
    out = torch.empty(N, dtype=torch.float32, device=mu.device)
    S = 0 if z is None else z.numel()
    with torch.cuda.device(mu.device):
        _lib.check(_lib.load().bb_acq_score(C.byref(acq), _ptr(mu), _ptr(var), N, _ptr(z), S, _ptr(out),
                                            _stream_ptr()), "bb_acq_score")
    return out


@_op_acq_score.register_fake
def _(mu, var, z, kind, params):
    return torch.empty_like(mu)


@torch.library.custom_op("baybe_b200::acq_score_joint", mutates_args=())
def _op_acq_score_joint(mu: torch.Tensor, var: torch.Tensor, cross: torch.Tensor, pend_mu: torch.Tensor,
                        pend_cov: torch.Tensor, z: torch.Tensor, kind: int,
                        params: list[float]) -> torch.Tensor:
    acq = AcqConfig.from_params(kind, params).to_c()
    N, P = cross.shape
    if z.dim() != 2 or z.shape[1] != P + 1:
        raise ValueError(f"base samples must be (S, {P + 1})")
    out = torch.empty(N, dtype=torch.float32, device=mu.device)
    with torch.cuda.device(mu.device):
        _lib.check(_lib.load().bb_acq_score_joint(C.byref(acq), _ptr(mu), _ptr(var), _ptr(cross), N,
                                                  _ptr(pend_mu), _ptr(pend_cov), P, _ptr(z), z.shape[0],
                                                  _ptr(out), _stream_ptr()), "bb_acq_score_joint")
    return out


@_op_acq_score_joint.register_fake
def _(mu, var, cross, pend_mu, pend_cov, z, kind, params):
    return torch.empty_like(mu)


@torch.library.custom_op("baybe_b200::acq_grad", mutates_args=())
def _op_acq_grad(x: torch.Tensor, pend_x: torch.Tensor | None, pend_beta: torch.Tensor | None,
                 pend_mu: torch.Tensor | None, pend_cov: torch.Tensor | None, z: torch.Tensor | None, handle: int,
                 kind: int, params: list[float]) -> tuple[torch.Tensor, torch.Tensor]:
    """``bb_acq_grad``: raw fp32 rows x [N, d] -> value [N], gradient [N, d]; with p pending points their rows
    pend_x [p, d] and ``pending_stats`` (beta [p, n_pad], mean [p], covariance [p, p]); z [S, 1 + p] (MC kinds)."""
    return _acq_grad_call("bb_acq_grad", x, pend_x, pend_beta, pend_mu, pend_cov, z, handle, kind, params)


@_op_acq_grad.register_fake
def _(x, pend_x, pend_beta, pend_mu, pend_cov, z, handle, kind, params):
    return x.new_empty(x.shape[0]), x.new_empty(x.shape)


@torch.library.custom_op("baybe_b200::acq_grad_large", mutates_args=())
def _op_acq_grad_large(x: torch.Tensor, pend_x: torch.Tensor | None, pend_beta: torch.Tensor | None,
                       pend_mu: torch.Tensor | None, pend_cov: torch.Tensor | None, z: torch.Tensor | None,
                       handle: int, kind: int, params: list[float]) -> tuple[torch.Tensor, torch.Tensor]:
    """``bb_acq_grad_large``: ``acq_grad`` for every single-task model (n_pad up to 1024, wide-feature or not)."""
    return _acq_grad_call("bb_acq_grad_large", x, pend_x, pend_beta, pend_mu, pend_cov, z, handle, kind, params)


@_op_acq_grad_large.register_fake
def _(x, pend_x, pend_beta, pend_mu, pend_cov, z, handle, kind, params):
    return x.new_empty(x.shape[0]), x.new_empty(x.shape)


def _acq_grad_call(entry: str, x, pend_x, pend_beta, pend_mu, pend_cov, z, handle, kind, params):
    """The body of the ``acq_grad`` and ``acq_grad_large`` ops: the two C entry points take the same arguments."""
    gp = _gp(handle)
    acq = AcqConfig.from_params(kind, params).to_c()
    N = x.shape[0]
    if x.dim() != 2 or x.shape[1] != gp.d or x.dtype != torch.float32 or not x.is_contiguous():
        raise ValueError(f"rows must be a contiguous float32 (N, {gp.d}) tensor")
    P = 0 if pend_x is None else pend_x.shape[0]
    if z is not None and (z.dim() != 2 or z.shape[1] != P + 1):
        raise ValueError(f"base samples must be (S, {P + 1})")
    value = torch.empty(N, dtype=torch.float32, device=x.device)
    grad = torch.empty((N, gp.d), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(getattr(_lib.load(), entry)(C.byref(gp.model), C.byref(acq), _ptr(x), N, P, _ptr(pend_x),
                                               _ptr(pend_beta), _ptr(pend_mu), _ptr(pend_cov), _ptr(z),
                                               0 if z is None else z.shape[0], _ptr(value), _ptr(grad),
                                               _stream_ptr()),
                   entry)
    return value, grad


def acq_grad_op(model: _lib.Model):
    """The gradient op ``DeviceGP.value_and_grad`` runs on a model: ``acq_grad`` (``bb_acq_grad``, one warp per point)
    for models that are not wide and have n_pad <= ``GRAD_MAX_NPAD``, ``acq_grad_large`` (``bb_acq_grad_large``, one
    CTA per point) for the rest.  Both compute the same function; task models are rejected by either."""
    if not model.wide and model.n_pad <= _lib.GRAD_MAX_NPAD:
        return torch.ops.baybe_b200.acq_grad
    return torch.ops.baybe_b200.acq_grad_large


def _check_keep(keep: torch.Tensor | None, N: int) -> None:
    if keep is not None and (keep.dtype != torch.uint8 or keep.numel() != N or not keep.is_contiguous()):
        raise ValueError("keep mask must be a contiguous uint8 tensor with one entry per candidate")


def _score_and_key(N: int, want_scores: bool, device) -> tuple[torch.Tensor, torch.Tensor]:
    """The outputs of a scoring op: scores [N] (empty without `want_scores`) and the packed best key, initialised on
    the current stream (called under ``torch.cuda.device(device)``)."""
    score = torch.empty(N if want_scores else 0, dtype=torch.float32, device=device)
    key = torch.empty(1, dtype=torch.int64, device=device)
    _lib.check(_lib.load().bb_best_init(_ptr(key), _stream_ptr()), "bb_best_init")
    return score, key


@torch.library.custom_op("baybe_b200::score_fused", mutates_args=())
def _op_score_fused(x: torch.Tensor, keep: torch.Tensor | None, z: torch.Tensor | None, handle: int,
                    kind: int, params: list[float], index_offset: int,
                    want_scores: bool) -> tuple[torch.Tensor, torch.Tensor]:
    gp = _gp(handle)
    acq = AcqConfig.from_params(kind, params).to_c()
    lay, ld = _layout_of(x)
    N = x.shape[0]
    _check_keep(keep, N)
    S = 0 if z is None else z.numel()
    lib = _lib.load()
    with torch.cuda.device(x.device):
        score, key = _score_and_key(N, want_scores, x.device)
        _lib.check(lib.bb_score_fused(C.byref(gp.model), C.byref(acq), _ptr(x), lay, N, ld, _ptr(keep),
                                      _ptr(z), S, _ptr(score) if want_scores else None, _ptr(key),
                                      index_offset, _stream_ptr()), "bb_score_fused")
    return score, key


@_op_score_fused.register_fake
def _(x, keep, z, handle, kind, params, index_offset, want_scores):
    return (x.new_empty(x.shape[0] if want_scores else 0, dtype=torch.float32),
            x.new_empty(1, dtype=torch.int64))


@torch.library.custom_op("baybe_b200::hvi_score", mutates_args=())
def _op_hvi_score(mu: torch.Tensor, var: torch.Tensor, cross: torch.Tensor | None, linv: torch.Tensor | None,
                  w: torch.Tensor | None, z: torch.Tensor, lower: torch.Tensor, upper: torch.Tensor,
                  n_cells: torch.Tensor, keep: torch.Tensor | None, kind: int, params: list[float],
                  obj_scale: list[float], obj_shift: list[float], index_offset: int,
                  want_scores: bool) -> tuple[torch.Tensor, torch.Tensor]:
    """``bb_hvi_score``: mu/var [M, N]; with P pending points cross [M, N, P], linv [M, P, P] (L_PP^-1), w [M, S, P];
    z [S, M(1+P)]; cells lower/upper [n_dec, C, M] float32 with counts n_cells [n_dec] int32."""
    acq = AcqConfig.from_params(kind, params).to_c()
    M, N = mu.shape
    P = 0 if cross is None else cross.shape[2]
    S = z.shape[0]
    if z.dim() != 2 or z.shape[1] != M * (1 + P):
        raise ValueError(f"base samples must be (S, {M * (1 + P)})")
    if lower.shape != upper.shape or lower.dim() != 3 or lower.shape[2] != M or n_cells.numel() != lower.shape[0] \
            or n_cells.dtype != torch.int32 or lower.shape[0] != (1 if P == 0 else S):
        raise ValueError("cells must be lower/upper [n_dec, C, M] with n_cells [n_dec] (n_dec = 1 or S)")
    _check_keep(keep, N)
    fa = (C.c_float * M)(*obj_scale)
    fb = (C.c_float * M)(*obj_shift)
    lib = _lib.load()
    with torch.cuda.device(mu.device):
        score, key = _score_and_key(N, want_scores, mu.device)
        _lib.check(lib.bb_hvi_score(C.byref(acq), M, fa, fb, N, _ptr(mu), _ptr(var), P, _ptr(cross), _ptr(linv),
                                    _ptr(w), _ptr(z), S, _ptr(lower), _ptr(upper), _ptr(n_cells), lower.shape[1],
                                    _ptr(keep), _ptr(score) if want_scores else None, _ptr(key), int(index_offset),
                                    _stream_ptr()), "bb_hvi_score")
    return score, key


@_op_hvi_score.register_fake
def _(mu, var, cross, linv, w, z, lower, upper, n_cells, keep, kind, params, obj_scale, obj_shift, index_offset,
      want_scores):
    return (mu.new_empty(mu.shape[1] if want_scores else 0, dtype=torch.float32), mu.new_empty(1, dtype=torch.int64))


@torch.library.custom_op("baybe_b200::hvi_decompose", mutates_args=())
def _op_hvi_decompose(points: torch.Tensor, n_points: torch.Tensor | None, ref: list[float],
                      cell_stride: int) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """``bb_hvi_decompose``: points [S, n, M] float32 (maximisation), n_points [S] int32 or None, ref [M] (float64
    on the host) -> lower/upper [S, cell_stride, M] float32, n_cells [S] int32 (above cell_stride: did not fit) and
    the hypervolume hv [S] float64 of every sample's points."""
    if points.dim() != 3 or points.dtype != torch.float32 or not points.is_contiguous():
        raise ValueError("points must be a contiguous float32 (S, n, M) tensor")
    S, n, M = points.shape
    if len(ref) != M:
        raise ValueError(f"one reference coordinate per target ({M})")
    if n_points is not None and (n_points.dtype != torch.int32 or n_points.numel() != S):
        raise ValueError(f"n_points must be an int32 tensor of {S} entries")
    dev = points.device
    lower = torch.empty((S, cell_stride, M), dtype=torch.float32, device=dev)
    upper = torch.empty((S, cell_stride, M), dtype=torch.float32, device=dev)
    n_cells = torch.empty(S, dtype=torch.int32, device=dev)
    hv = torch.empty(S, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().bb_hvi_decompose(M, (C.c_double * M)(*ref), S, n, _ptr(points), _ptr(n_points),
                                                int(cell_stride), _ptr(lower), _ptr(upper), _ptr(n_cells), _ptr(hv),
                                                _stream_ptr()), "bb_hvi_decompose")
    return lower, upper, n_cells, hv


@_op_hvi_decompose.register_fake
def _(points, n_points, ref, cell_stride):
    S, _, M = points.shape
    return (points.new_empty((S, cell_stride, M)), points.new_empty((S, cell_stride, M)),
            points.new_empty(S, dtype=torch.int32), points.new_empty(S, dtype=torch.float64))


@torch.library.custom_op("baybe_b200::joint_posterior", mutates_args=())
def _op_joint_posterior(x: torch.Tensor, handle: int, with_beta: bool) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """``bb_joint_posterior``: float64 mean [R] and covariance [R, R] of R raw fp32 rows [R, d]; with `with_beta`
    also beta = K^-1 k(X, rows) [R, n_pad] fp32 (the input ``posterior_cross`` takes for them), else a [0, n_pad]
    tensor."""
    gp = _gp(handle)
    R = x.shape[0]
    if x.dim() != 2 or x.shape[1] != gp.d or x.dtype != torch.float32 or not x.is_contiguous():
        raise ValueError(f"rows must be a contiguous float32 (R, {gp.d}) tensor")
    mu = torch.empty(R, dtype=torch.float64, device=x.device)
    cov = torch.empty((R, R), dtype=torch.float64, device=x.device)
    beta = torch.empty((R if with_beta else 0, gp.model.n_pad), dtype=torch.float32, device=x.device)
    ws = torch.empty(max(R, 1) * (gp.model.n_pad + gp.d), dtype=torch.float64, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().bb_joint_posterior(C.byref(gp.model), _ptr(x), R, _ptr(mu), _ptr(cov),
                                                  _ptr(beta) if with_beta else None, _ptr(ws), ws.numel(),
                                                  _stream_ptr()), "bb_joint_posterior")
    return mu, cov, beta


@_op_joint_posterior.register_fake
def _(x, handle, with_beta):
    R = x.shape[0]
    return (x.new_empty(R, dtype=torch.float64), x.new_empty((R, R), dtype=torch.float64),
            x.new_empty((R if with_beta else 0, _gp(handle).model.n_pad), dtype=torch.float32))


@torch.library.custom_op("baybe_b200::nei_score", mutates_args=())
def _op_nei_score(mu: torch.Tensor, var: torch.Tensor, cross: torch.Tensor | None, linv: torch.Tensor | None,
                  w: torch.Tensor | None, z: torch.Tensor, g: torch.Tensor, batch_terms: torch.Tensor | None,
                  keep: torch.Tensor | None, log_nei: bool, params: list[float], index_offset: int,
                  want_scores: bool) -> tuple[torch.Tensor, torch.Tensor]:
    """``bb_nei_score``: mu/var [N]; with |C| conditioning points cross [N, |C|], linv [|C|, |C|] (L_C^-1) and
    w [|C|, S] (sample-minor); z [S, 1 + |C|]; g [S]; batch_terms [S, Q] for the other Q points of a q-batch.
    params = [obj_scale, obj_shift, tau_relu, tau_max]."""
    N = mu.shape[0]
    Cn = 0 if cross is None else cross.shape[1]
    S = z.shape[0]
    if z.dim() != 2 or z.shape[1] != Cn + 1:
        raise ValueError(f"base samples must be (S, {Cn + 1})")
    if g.numel() != S:
        raise ValueError(f"incumbents must be (S,) = ({S},)")
    if Cn and (linv is None or tuple(linv.shape) != (Cn, Cn) or w is None or tuple(w.shape) != (Cn, S)):
        raise ValueError(f"conditioning needs linv ({Cn}, {Cn}) and w ({Cn}, {S})")
    Q = 0 if batch_terms is None else batch_terms.shape[1]
    if Q and tuple(batch_terms.shape) != (S, Q):
        raise ValueError(f"batch terms must be (S, Q) = ({S}, {Q})")
    _check_keep(keep, N)
    a, b, tau_relu, tau_max = (float(v) for v in params)
    lib = _lib.load()
    with torch.cuda.device(mu.device):
        score, key = _score_and_key(N, want_scores, mu.device)
        _lib.check(lib.bb_nei_score(int(log_nei), a, b, tau_relu, tau_max, N, _ptr(mu), _ptr(var), Cn, _ptr(cross),
                                    _ptr(linv), _ptr(w), _ptr(z), S, _ptr(g), Q, _ptr(batch_terms), _ptr(keep),
                                    _ptr(score) if want_scores else None, _ptr(key), int(index_offset),
                                    _stream_ptr()), "bb_nei_score")
    return score, key


@_op_nei_score.register_fake
def _(mu, var, cross, linv, w, z, g, batch_terms, keep, log_nei, params, index_offset, want_scores):
    return (mu.new_empty(mu.shape[0] if want_scores else 0, dtype=torch.float32), mu.new_empty(1, dtype=torch.int64))


_NIPV_WS_CAP = 768 << 20  # workspace of bb_nipv_score: rows are processed in blocks that fit it


def nipv_model_terms(gp: DeviceGP) -> tuple[list[float], float]:
    """The likelihood noise per task (standardised, floored at 1e-4) and the largest prior variance over the tasks
    (standardised) of a model: what ``bb_nipv_score`` takes besides the model."""
    scale = 1.0 if gp.outputscale is None else gp.outputscale
    diag = np.ones(1) if gp.task_covar is None else np.diag(gp.task_covar)
    return [max(float(v), 1e-4) for v in gp.noise], float(scale * diag.max())


@torch.library.custom_op("baybe_b200::nipv_score", mutates_args=())
def _op_nipv_score(x: torch.Tensor, xm: torch.Tensor, var: torch.Tensor, cross_x: torch.Tensor | None,
                   cross_m: torch.Tensor | None, linv: torch.Tensor | None, keep: torch.Tensor | None, handle: int,
                   index_offset: int, want_scores: bool) -> tuple[torch.Tensor, torch.Tensor]:
    """``bb_nipv_score``: candidates x [N, d] and integration points xm [M, d] (raw fp32 rows), the candidates'
    posterior variance var [N]; with |C| conditioning points cross_x [N, |C|], cross_m [M, |C|] and linv [|C|, |C|]
    (L_C^-1 of K_D(C,C) + noise, original units).  Scores: IVR(x) in original units."""
    gp = _gp(handle)
    N, M = x.shape[0], xm.shape[0]
    for name, t, rows in (("x", x, N), ("xm", xm, M)):
        if t.dim() != 2 or t.shape[1] != gp.d or t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError(f"{name} must be a contiguous float32 ({rows}, {gp.d}) tensor")
    Cn = 0 if cross_x is None else cross_x.shape[1]
    if Cn and (cross_m is None or tuple(cross_m.shape) != (M, Cn) or linv is None or tuple(linv.shape) != (Cn, Cn)):
        raise ValueError(f"conditioning needs cross_m ({M}, {Cn}) and linv ({Cn}, {Cn})")
    _check_keep(keep, N)
    f32 = lambda t: None if t is None else t.to(torch.float32).contiguous()  # noqa: E731
    var, cross_x, cross_m, linv = f32(var), f32(cross_x), f32(cross_m), f32(linv)
    noise, prior_var = nipv_model_terms(gp)
    r_pad = -(-(gp.n + Cn) // 64) * 64
    row_bytes = 4 * r_pad + 4 * gp.d + 12
    ws_bytes = min(_NIPV_WS_CAP, (N + M + 256) * row_bytes)
    lib = _lib.load()
    with torch.cuda.device(x.device):
        score, key = _score_and_key(N, want_scores, x.device)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=x.device)
        _lib.check(lib.bb_nipv_score(C.byref(gp.model), (C.c_float * len(noise))(*noise), prior_var, _ptr(x), N,
                                     _ptr(xm), M, _ptr(var), Cn, _ptr(cross_x), _ptr(cross_m), _ptr(linv),
                                     _ptr(keep), _ptr(score) if want_scores else None, _ptr(key), int(index_offset),
                                     _ptr(ws), ws_bytes, _stream_ptr()), "bb_nipv_score")
    return score, key


@_op_nipv_score.register_fake
def _(x, xm, var, cross_x, cross_m, linv, keep, handle, index_offset, want_scores):
    return (x.new_empty(x.shape[0] if want_scores else 0, dtype=torch.float32), x.new_empty(1, dtype=torch.int64))


def nipv_image_numel(gp: DeviceGP, M: int, n_cond: int) -> int:
    """Floats of ``bb_nipv_phi``'s image, (n + n_cond + d) M; raises ``NotImplementedError`` above
    ``_lib.NIPV_IMAGE_CAP`` bytes."""
    numel = (gp.n + n_cond + gp.d) * M
    if 4 * numel > _lib.NIPV_IMAGE_CAP:
        raise NotImplementedError(
            f"qNIPV's gradient path keeps an image of (n + |C| + d) x M = {gp.n + n_cond + gp.d} x {M} fp32 values on "
            f"the device, above its cap of {_lib.NIPV_IMAGE_CAP >> 30} GiB: use fewer integration points")
    return numel


@torch.library.custom_op("baybe_b200::nipv_phi", mutates_args=())
def _op_nipv_phi(xm: torch.Tensor, cross_m: torch.Tensor | None, linv: torch.Tensor | None,
                 handle: int) -> torch.Tensor:
    """``bb_nipv_phi``: integration points xm [M, d] (raw fp32 rows); with |C| conditioning points cross_m [M, |C|] and
    linv [|C|, |C|] as ``nipv_score``.  Returns the image [(n + |C| + d) * M] fp32."""
    gp = _gp(handle)
    M = xm.shape[0]
    if xm.dim() != 2 or xm.shape[1] != gp.d or xm.dtype != torch.float32 or not xm.is_contiguous():
        raise ValueError(f"xm must be a contiguous float32 ({M}, {gp.d}) tensor")
    Cn = 0 if cross_m is None else cross_m.shape[1]
    if Cn and (tuple(cross_m.shape) != (M, Cn) or linv is None or tuple(linv.shape) != (Cn, Cn)):
        raise ValueError(f"conditioning needs cross_m ({M}, {Cn}) and linv ({Cn}, {Cn})")
    f32 = lambda t: None if t is None else t.to(torch.float32).contiguous()  # noqa: E731
    cross_m, linv = f32(cross_m), f32(linv)
    img = torch.empty(nipv_image_numel(gp, M, Cn), dtype=torch.float32, device=xm.device)
    with torch.cuda.device(xm.device):
        _lib.check(_lib.load().bb_nipv_phi(C.byref(gp.model), _ptr(xm), M, Cn, _ptr(cross_m), _ptr(linv), _ptr(img),
                                           _stream_ptr()), "bb_nipv_phi")
    return img


@_op_nipv_phi.register_fake
def _(xm, cross_m, linv, handle):
    gp = _gp(handle)
    Cn = 0 if cross_m is None else cross_m.shape[1]
    return xm.new_empty((gp.n + Cn + gp.d) * xm.shape[0])


@torch.library.custom_op("baybe_b200::nipv_grad", mutates_args=())
def _op_nipv_grad(x: torch.Tensor, img: torch.Tensor, M: int, cond_x: torch.Tensor | None,
                  cond_beta: torch.Tensor | None, linv: torch.Tensor | None,
                  handle: int) -> tuple[torch.Tensor, torch.Tensor]:
    """``bb_nipv_grad``: points x [P, d] (raw fp32 rows), ``nipv_phi``'s image of M integration points; with |C|
    conditioning points their raw rows cond_x [|C|, d], beta [|C|, n_pad] (``bb_joint_posterior``) and linv
    [|C|, |C|].  Returns IVR [P] (original units, as ``nipv_score``) and its gradient [P, d]."""
    gp = _gp(handle)
    P = x.shape[0]
    if x.dim() != 2 or x.shape[1] != gp.d or x.dtype != torch.float32 or not x.is_contiguous():
        raise ValueError(f"x must be a contiguous float32 ({P}, {gp.d}) tensor")
    Cn = 0 if cond_x is None else cond_x.shape[0]
    if img.numel() != (gp.n + Cn + gp.d) * M:
        raise ValueError(f"the image must hold (n + |C| + d) * M = {(gp.n + Cn + gp.d) * M} values")
    if Cn and (tuple(cond_x.shape) != (Cn, gp.d) or cond_beta is None or cond_beta.shape[0] != Cn
               or linv is None or tuple(linv.shape) != (Cn, Cn)):
        raise ValueError(f"conditioning needs cond_x ({Cn}, {gp.d}), beta ({Cn}, n_pad) and linv ({Cn}, {Cn})")
    f32 = lambda t: None if t is None else t.to(torch.float32).contiguous()  # noqa: E731
    cond_x, cond_beta, linv = f32(cond_x), f32(cond_beta), f32(linv)
    noise, prior_var = nipv_model_terms(gp)
    value = torch.empty(P, dtype=torch.float32, device=x.device)
    grad = torch.empty((P, gp.d), dtype=torch.float32, device=x.device)
    if P == 0:
        return value, grad
    ws_bytes = _lib.nipv_grad_ws_bytes(P, M, gp.n, Cn, gp.d)
    with torch.cuda.device(x.device):
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        _lib.check(_lib.load().bb_nipv_grad(C.byref(gp.model), (C.c_float * len(noise))(*noise), prior_var, _ptr(x),
                                            P, _ptr(img), M, Cn, _ptr(cond_x), _ptr(cond_beta), _ptr(linv),
                                            _ptr(value), _ptr(grad), _ptr(ws), ws_bytes, _stream_ptr()),
                   "bb_nipv_grad")
    return value, grad


@_op_nipv_grad.register_fake
def _(x, img, M, cond_x, cond_beta, linv, handle):
    return x.new_empty(x.shape[0]), x.new_empty(x.shape)


@torch.library.custom_op("baybe_b200::parego_score", mutates_args=())
def _op_parego_score(mu: torch.Tensor, var: torch.Tensor, cross: torch.Tensor | None, linv: torch.Tensor | None,
                     w: torch.Tensor | None, z: torch.Tensor, g: torch.Tensor, batch_terms: torch.Tensor | None,
                     keep: torch.Tensor | None, weight: list[float], offset: list[float], params: list[float],
                     index_offset: int, want_scores: bool) -> tuple[torch.Tensor, torch.Tensor]:
    """``bb_parego_score``: mu/var [M, N]; with |C| conditioning points cross [M, N, |C|], linv [M, |C|, |C|]
    (L_C^-1 per target) and w [M, |C|, S] (sample-minor); z [S, M(1 + |C|)]; g [S]; batch_terms [S, Q] for the other
    Q points of a q-batch; p_m = weight[m] y_m + offset[m]; params = [alpha, tau_relu, tau_max]."""
    M, N = mu.shape
    Cn = 0 if cross is None else cross.shape[2]
    S = z.shape[0]
    if z.dim() != 2 or z.shape[1] != M * (Cn + 1):
        raise ValueError(f"base samples must be (S, {M * (Cn + 1)})")
    if len(weight) != M or len(offset) != M:
        raise ValueError(f"one scalarisation weight and offset per target ({M})")
    if g.numel() != S:
        raise ValueError(f"incumbents must be (S,) = ({S},)")
    if Cn and (linv is None or tuple(linv.shape) != (M, Cn, Cn) or w is None or tuple(w.shape) != (M, Cn, S)):
        raise ValueError(f"conditioning needs linv ({M}, {Cn}, {Cn}) and w ({M}, {Cn}, {S})")
    Q = 0 if batch_terms is None else batch_terms.shape[1]
    if Q and tuple(batch_terms.shape) != (S, Q):
        raise ValueError(f"batch terms must be (S, Q) = ({S}, {Q})")
    _check_keep(keep, N)
    alpha, tau_relu, tau_max = (float(v) for v in params)
    fw = (C.c_float * M)(*weight)
    fv = (C.c_float * M)(*offset)
    lib = _lib.load()
    with torch.cuda.device(mu.device):
        score, key = _score_and_key(N, want_scores, mu.device)
        _lib.check(lib.bb_parego_score(M, fw, fv, alpha, tau_relu, tau_max, N, _ptr(mu), _ptr(var), Cn, _ptr(cross),
                                       _ptr(linv), _ptr(w), _ptr(z), S, _ptr(g), Q, _ptr(batch_terms), _ptr(keep),
                                       _ptr(score) if want_scores else None, _ptr(key), int(index_offset),
                                       _stream_ptr()), "bb_parego_score")
    return score, key


@_op_parego_score.register_fake
def _(mu, var, cross, linv, w, z, g, batch_terms, keep, weight, offset, params, index_offset, want_scores):
    return (mu.new_empty(mu.shape[1] if want_scores else 0, dtype=torch.float32), mu.new_empty(1, dtype=torch.int64))


def objective_struct(n_targets: int, scalarizer: int, programs, weights) -> _lib.Objective:
    """``bb_objective`` from per-target programs [(opcode, (arg0, arg1, arg2)), ...] (baybe_b200/objectives.py)."""
    obj = _lib.Objective()
    obj.n_targets, obj.scalarizer = int(n_targets), int(scalarizer)
    if len(programs) > _lib.OBJ_MAX_TARGETS:
        raise ValueError(f"at most {_lib.OBJ_MAX_TARGETS} target programs")
    for m, prog in enumerate(programs):
        if len(prog) > _lib.OBJ_MAX_OPS:
            raise ValueError(f"at most {_lib.OBJ_MAX_OPS} ops per target")
        obj.n_ops[m] = len(prog)
        obj.weight[m] = float(weights[m])
        for i, (op, args) in enumerate(prog):
            obj.prog[m][i].op = int(op)
            for k, v in enumerate(args):
                obj.prog[m][i].arg[k] = float(v)
    return obj


@torch.library.custom_op("baybe_b200::objective_score", mutates_args=())
def _op_objective_score(mu: torch.Tensor, var: torch.Tensor, cross: torch.Tensor | None, linv: torch.Tensor | None,
                        w: torch.Tensor | None, pend_terms: torch.Tensor | None, z: torch.Tensor | None,
                        keep: torch.Tensor | None, kind: int, params: list[float], scalarizer: int,
                        ops: list[int], args: list[float], n_ops: list[int], weights: list[float], index_offset: int,
                        want_scores: bool) -> tuple[torch.Tensor, torch.Tensor]:
    """``bb_objective_score``: mu/var [M, N]; with P pending points cross [M, N, P], linv [M, P, P], w [M, S, P] and
    pend_terms [S, P]; z [S, M(1+P)] (None for analytic kinds).  The programs come flattened: target m owns n_ops[m]
    consecutive entries of ops (opcodes) and of args (three floats each)."""
    acq = AcqConfig.from_params(kind, params).to_c()
    M, N = mu.shape
    P = 0 if cross is None else cross.shape[2]
    S = 0 if z is None else z.shape[0]
    if z is not None and (z.dim() != 2 or z.shape[1] != M * (1 + P)):
        raise ValueError(f"base samples must be (S, {M * (1 + P)})")
    if P and (pend_terms is None or tuple(pend_terms.shape) != (S, P)):
        raise ValueError(f"pending terms must be (S, P) = ({S}, {P})")
    _check_keep(keep, N)
    progs, k = [], 0
    for n in n_ops:
        progs.append([(ops[k + i], args[3 * (k + i): 3 * (k + i) + 3]) for i in range(n)])
        k += n
    obj = objective_struct(M, scalarizer, progs, weights)
    lib = _lib.load()
    with torch.cuda.device(mu.device):
        score, key = _score_and_key(N, want_scores, mu.device)
        _lib.check(lib.bb_objective_score(C.byref(acq), C.byref(obj), N, _ptr(mu), _ptr(var), P, _ptr(cross),
                                          _ptr(linv), _ptr(w), _ptr(pend_terms), _ptr(z), S, _ptr(keep),
                                          _ptr(score) if want_scores else None, _ptr(key), int(index_offset),
                                          _stream_ptr()), "bb_objective_score")
    return score, key


@_op_objective_score.register_fake
def _(mu, var, cross, linv, w, pend_terms, z, keep, kind, params, scalarizer, ops, args, n_ops, weights, index_offset,
      want_scores):
    return (mu.new_empty(mu.shape[1] if want_scores else 0, dtype=torch.float32), mu.new_empty(1, dtype=torch.int64))


def _unflatten_programs(ops: list[int], args: list[float], n_ops: list[int]) -> list:
    progs, k = [], 0
    for n in n_ops:
        progs.append([(ops[k + i], args[3 * (k + i): 3 * (k + i) + 3]) for i in range(n)])
        k += n
    return progs


@torch.library.custom_op("baybe_b200::objective_grad", mutates_args=())
def _op_objective_grad(x: torch.Tensor, handles: list[int], pend_x: torch.Tensor | None, betas: list[torch.Tensor],
                       linv: torch.Tensor | None, w: torch.Tensor | None, pend_terms: torch.Tensor | None,
                       z: torch.Tensor | None, kind: int, params: list[float], scalarizer: int, ops: list[int],
                       args: list[float], n_ops: list[int], weights: list[float]) -> tuple[torch.Tensor, torch.Tensor]:
    """``bb_objective_grad``: raw fp32 rows x [N, d] of the models `handles` (one per target) -> value [N], gradient
    [N, d].  With P pending points their rows pend_x [P, d], one beta [P, n_pad] per model (``pending_stats``), linv
    [M, P, P], w [M, S, P] and pend_terms [S, P] (as ``objective_score``); z [S, M(1+P)] (None for analytic kinds)."""
    return _objective_grad_call("bb_objective_grad", x, handles, pend_x, betas, linv, w, pend_terms, z, kind, params,
                                scalarizer, ops, args, n_ops, weights)


@_op_objective_grad.register_fake
def _(x, handles, pend_x, betas, linv, w, pend_terms, z, kind, params, scalarizer, ops, args, n_ops, weights):
    return x.new_empty(x.shape[0]), x.new_empty(x.shape)


@torch.library.custom_op("baybe_b200::objective_grad_large", mutates_args=())
def _op_objective_grad_large(x: torch.Tensor, handles: list[int], pend_x: torch.Tensor | None,
                             betas: list[torch.Tensor], linv: torch.Tensor | None, w: torch.Tensor | None,
                             pend_terms: torch.Tensor | None, z: torch.Tensor | None, kind: int, params: list[float],
                             scalarizer: int, ops: list[int], args: list[float], n_ops: list[int],
                             weights: list[float]) -> tuple[torch.Tensor, torch.Tensor]:
    """``bb_objective_grad_large``: ``objective_grad`` for every mix of single-task models (n_pad up to 1024,
    wide-feature or not)."""
    return _objective_grad_call("bb_objective_grad_large", x, handles, pend_x, betas, linv, w, pend_terms, z, kind,
                                params, scalarizer, ops, args, n_ops, weights)


@_op_objective_grad_large.register_fake
def _(x, handles, pend_x, betas, linv, w, pend_terms, z, kind, params, scalarizer, ops, args, n_ops, weights):
    return x.new_empty(x.shape[0]), x.new_empty(x.shape)


def _objective_grad_call(entry: str, x, handles, pend_x, betas, linv, w, pend_terms, z, kind, params, scalarizer, ops,
                         args, n_ops, weights):
    """The body of the ``objective_grad`` and ``objective_grad_large`` ops: the two C entry points take the same
    arguments."""
    gps = [_gp(h) for h in handles]
    M, N = len(gps), x.shape[0]
    if x.dim() != 2 or x.shape[1] != gps[0].d or x.dtype != torch.float32 or not x.is_contiguous():
        raise ValueError(f"rows must be a contiguous float32 (N, {gps[0].d}) tensor")
    P = 0 if pend_x is None else pend_x.shape[0]
    if z is not None and (z.dim() != 2 or z.shape[1] != M * (1 + P)):
        raise ValueError(f"base samples must be (S, {M * (1 + P)})")
    if P and len(betas) != M:
        raise ValueError(f"{P} pending points need one beta per model ({M})")
    acq = AcqConfig.from_params(kind, params).to_c()
    obj = objective_struct(M, scalarizer, _unflatten_programs(ops, args, n_ops), weights)
    models = (C.POINTER(_lib.Model) * M)(*(C.pointer(gp.model) for gp in gps))
    beta_ptrs = (C.c_void_p * M)(*((b.data_ptr() for b in betas) if P else [None] * M))
    value = torch.empty(N, dtype=torch.float32, device=x.device)
    grad = torch.empty((N, x.shape[1]), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(getattr(_lib.load(), entry)(models, M, C.byref(acq), C.byref(obj), _ptr(x), N, P, _ptr(pend_x),
                                               beta_ptrs if P else None, _ptr(linv), _ptr(w), _ptr(pend_terms),
                                               _ptr(z), 0 if z is None else z.shape[0], _ptr(value), _ptr(grad),
                                               _stream_ptr()), entry)
    return value, grad


def objective_grad_op(models):
    """The gradient op ``ObjectiveScorer.value_and_grad`` runs on the models of an objective's targets (one each):
    ``objective_grad`` (``bb_objective_grad``, one warp per point) when every model is not wide and has n_pad <=
    ``GRAD_MAX_NPAD``, ``objective_grad_large`` (``bb_objective_grad_large``, one CTA per point) otherwise.  Both
    compute the same function; task models are rejected by either."""
    if all(not m.wide and m.n_pad <= _lib.GRAD_MAX_NPAD for m in models):
        return torch.ops.baybe_b200.objective_grad
    return torch.ops.baybe_b200.objective_grad_large


@torch.library.custom_op("baybe_b200::hvi_grad", mutates_args=())
def _op_hvi_grad(x: torch.Tensor, handles: list[int], pend_x: torch.Tensor | None, betas: list[torch.Tensor],
                 linv: torch.Tensor | None, w: torch.Tensor | None, z: torch.Tensor, lower: torch.Tensor,
                 upper: torch.Tensor, n_cells: torch.Tensor, kind: int, params: list[float], obj_scale: list[float],
                 obj_shift: list[float]) -> tuple[torch.Tensor, torch.Tensor]:
    """``bb_hvi_grad``: raw fp32 rows x [N, d] of the models `handles` (one per target) -> value [N] (what
    ``hvi_score`` scores), gradient [N, d].  With P pending points their rows pend_x [P, d], one beta [P, n_pad] per
    model (``pending_stats``), linv [M, P, P] and w [M, S, P]; z [S, M(1+P)]; cells lower/upper [n_dec, C, M] float32
    with counts n_cells [n_dec] int32 (n_dec = 1 without pending points, else S), as ``hvi_score``."""
    gps = [_gp(h) for h in handles]
    M, N = len(gps), x.shape[0]
    if x.dim() != 2 or x.shape[1] != gps[0].d or x.dtype != torch.float32 or not x.is_contiguous():
        raise ValueError(f"rows must be a contiguous float32 (N, {gps[0].d}) tensor")
    P = 0 if pend_x is None else pend_x.shape[0]
    S = z.shape[0]
    if z.dim() != 2 or z.shape[1] != M * (1 + P):
        raise ValueError(f"base samples must be (S, {M * (1 + P)})")
    if P and len(betas) != M:
        raise ValueError(f"{P} pending points need one beta per model ({M})")
    if lower.shape != upper.shape or lower.dim() != 3 or lower.shape[2] != M or n_cells.numel() != lower.shape[0] \
            or n_cells.dtype != torch.int32 or lower.shape[0] != (1 if P == 0 else S):
        raise ValueError("cells must be lower/upper [n_dec, C, M] with n_cells [n_dec] (n_dec = 1 or S)")
    acq = AcqConfig.from_params(kind, params).to_c()
    models = (C.POINTER(_lib.Model) * M)(*(C.pointer(gp.model) for gp in gps))
    beta_ptrs = (C.c_void_p * M)(*((b.data_ptr() for b in betas) if P else [None] * M))
    fa = (C.c_float * M)(*obj_scale)
    fb = (C.c_float * M)(*obj_shift)
    value = torch.empty(N, dtype=torch.float32, device=x.device)
    grad = torch.empty((N, x.shape[1]), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().bb_hvi_grad(models, M, C.byref(acq), fa, fb, _ptr(x), N, P, _ptr(pend_x),
                                           beta_ptrs if P else None, _ptr(linv), _ptr(w), _ptr(z), S, _ptr(lower),
                                           _ptr(upper), _ptr(n_cells), lower.shape[1], _ptr(value), _ptr(grad),
                                           _stream_ptr()), "bb_hvi_grad")
    return value, grad


@_op_hvi_grad.register_fake
def _(x, handles, pend_x, betas, linv, w, z, lower, upper, n_cells, kind, params, obj_scale, obj_shift):
    return x.new_empty(x.shape[0]), x.new_empty(x.shape)


@torch.library.custom_op("baybe_b200::argmax", mutates_args=())
def _op_argmax(score: torch.Tensor, keep: torch.Tensor | None, index_offset: int) -> torch.Tensor:
    key = torch.empty(1, dtype=torch.int64, device=score.device)
    lib = _lib.load()
    with torch.cuda.device(score.device):
        _lib.check(lib.bb_best_init(_ptr(key), _stream_ptr()), "bb_best_init")
        _lib.check(lib.bb_argmax(_ptr(score), _ptr(keep), score.numel(), index_offset, _ptr(key),
                                 _stream_ptr()), "bb_argmax")
    return key


@_op_argmax.register_fake
def _(score, keep, index_offset):
    return score.new_empty(1, dtype=torch.int64)


@torch.library.custom_op("baybe_b200::best_decode", mutates_args=())
def _op_best_decode(key: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    raw = torch.empty(2, dtype=torch.int64, device=key.device)  # sizeof(bb_best) == 16
    with torch.cuda.device(key.device):
        _lib.check(_lib.load().bb_best_decode(_ptr(key), _ptr(raw), _stream_ptr()), "bb_best_decode")
    val = raw[:1].view(torch.float32)[:1].clone()
    return val, raw[1:2].clone()


@_op_best_decode.register_fake
def _(key):
    return key.new_empty(1, dtype=torch.float32), key.new_empty(1, dtype=torch.int64)


@torch.library.custom_op("baybe_b200::topk", mutates_args=())
def _op_topk(score: torch.Tensor, keep: torch.Tensor | None, k: int) -> tuple[torch.Tensor, torch.Tensor]:
    N = score.numel()
    vals = torch.empty(k, dtype=torch.float32, device=score.device)
    idx = torch.empty(k, dtype=torch.int64, device=score.device)
    mask = torch.empty(N, dtype=torch.uint8, device=score.device)
    key = torch.empty(1, dtype=torch.int64, device=score.device)
    with torch.cuda.device(score.device):
        _lib.check(_lib.load().bb_topk(_ptr(score), _ptr(keep), N, k, _ptr(vals), _ptr(idx), _ptr(mask),
                                       _ptr(key), _stream_ptr()), "bb_topk")
    return vals, idx


@_op_topk.register_fake
def _(score, keep, k):
    return score.new_empty(k, dtype=torch.float32), score.new_empty(k, dtype=torch.int64)
