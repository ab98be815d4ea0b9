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
        if self.kind not in _lib.ACQ_KIND and self.kind not in _lib.NEI_KINDS:
            raise ValueError(f"unsupported acquisition function {self.kind!r}")

    @property
    def is_mc(self) -> bool:
        return self.kind in _lib.MC_KINDS or self.kind in _lib.NEI_KINDS

    def to_c(self) -> _lib.AcqSpec:
        if self.kind in _lib.NEI_KINDS:
            raise NotImplementedError(f"{self.kind} is evaluated by baybe_b200.hybrid.NeiScorer, not by the fused kernels")
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
    index).  Used by the CPU tests of the sharded arg-max protocol."""
    import struct

    u = struct.unpack("<i", struct.pack("<f", score))[0]
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


@torch.library.custom_op("baybe_b200::score_fused", mutates_args=())
def _op_score_fused(x: torch.Tensor, keep: torch.Tensor | None, z: torch.Tensor | None, handle: int,
                    kind: int, params: list[float], index_offset: int,
                    want_scores: bool) -> tuple[torch.Tensor, torch.Tensor]:
    gp = _gp(handle)
    acq = AcqConfig.from_params(kind, params).to_c()
    lay, ld = _layout_of(x)
    N = x.shape[0]
    score = torch.empty(N if want_scores else 0, dtype=torch.float32, device=x.device)
    key = torch.empty(1, dtype=torch.int64, device=x.device)
    if keep is not None and (keep.dtype != torch.uint8 or keep.numel() != N or not keep.is_contiguous()):
        raise ValueError("keep mask must be a contiguous uint8 tensor with one entry per candidate")
    S = 0 if z is None else z.numel()
    lib = _lib.load()
    with torch.cuda.device(x.device):
        _lib.check(lib.bb_best_init(_ptr(key), _stream_ptr()), "bb_best_init")
        _lib.check(lib.bb_score_fused(C.byref(gp.model), C.byref(acq), _ptr(x), lay, N, ld, _ptr(keep),
                                      _ptr(z), S, _ptr(score) if want_scores else None, _ptr(key),
                                      index_offset, _stream_ptr()), "bb_score_fused")
    return score, key


@_op_score_fused.register_fake
def _(x, keep, z, handle, kind, params, index_offset, want_scores):
    return (x.new_empty(x.shape[0] if want_scores else 0, dtype=torch.float32),
            x.new_empty(1, dtype=torch.int64))


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
