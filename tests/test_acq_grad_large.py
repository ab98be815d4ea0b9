"""CPU tests of ``bb_acq_grad_large``: its argument checks before any CUDA call, and the choice between it and
``bb_acq_grad`` (``engine.acq_grad_op``), on model structs filled by hand."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from baybe_b200.acquisition import AcqConfig
from baybe_b200.continuous import recommend_continuous_hybrid
from tests.continuous_oracle import OracleGradGP


@pytest.fixture(scope="module")
def lib():
    from baybe_b200 import _lib
    from baybe_b200.build import build

    build(verbose=False)
    return _lib.load()


def _fake(wide=False, task=False, n_pad=64):
    from tests.test_abi import _fake_model

    m = _fake_model(wide, 1)
    m.n = m.n_pad = n_pad
    if task:
        m.task_col = 0
    return m


@pytest.mark.parametrize("case, status, msg", [
    ("null model", "invalid", b"model struct"),
    ("abi mismatch", "invalid", b"ABI mismatch"),
    ("null spec", "invalid", b"spec is null"),
    ("kind -1", "invalid", b"single-target"),
    ("kind 11", "invalid", b"single-target"),
    ("task", "unsupported", b"task parameter"),
    ("n_pad 1088", "unsupported", b"n_pad=1088"),
    ("negative N", "invalid", b"negative point count"),
    ("pending analytic", "invalid", b"Monte Carlo"),
    ("33 pending", "invalid", b"n_pending=33"),
    ("S 0", "invalid", b"S=0"),
    ("S 1025", "invalid", b"S=1025"),
    ("null samples", "invalid", b"base samples"),
    ("null pending", "invalid", b"pending buffer"),
    ("null output", "invalid", b"null buffer"),
])
def test_acq_grad_large_rejects_bad_arguments_before_any_cuda_call(lib, case, status, msg):
    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    m = _fake(task=case == "task", n_pad=1088 if case == "n_pad 1088" else 512)
    if case == "abi mismatch":
        m.abi_version = _lib.ABI_VERSION + 1
    kind = {"kind -1": -1, "kind 11": 11, "pending analytic": _lib.ACQ_KIND["EI"]}.get(case, _lib.ACQ_KIND["qEI"])
    a = _lib.AcqSpec(kind=kind, obj_scale=1.0)
    buf = C.c_void_p(1 << 20)
    P = {"pending analytic": 1, "33 pending": 33, "null pending": 2}.get(case, 0)
    S = {"S 0": 0, "S 1025": 1025}.get(case, 64)
    z = None if case == "null samples" else buf
    pend = None if case == "null pending" else buf
    out = None if case == "null output" else buf
    N = -1 if case == "negative N" else 10
    rc = lib.bb_acq_grad_large(None if case == "null model" else C.byref(m),
                               None if case == "null spec" else C.byref(a), buf, N, P, pend, pend, pend, pend, z, S,
                               out, out, None)
    assert rc == {"invalid": _lib.BB_ERR_INVALID, "unsupported": _lib.BB_ERR_UNSUPPORTED}[status]
    assert msg in lib.bb_last_error()
    assert lib.bb_last_error().startswith(b"bb_acq_grad_large: ")


@pytest.mark.parametrize("wide, n_pad", [(False, 512), (False, 1024), (True, 128), (True, 1024)])
def test_acq_grad_large_takes_the_models_bb_acq_grad_rejects(lib, wide, n_pad):
    """Wide models and n_pad up to 1024 pass every check of bb_acq_grad_large (N = 0 returns before any CUDA call),
    where bb_acq_grad returns BB_ERR_UNSUPPORTED."""
    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    m = _fake(wide=wide, n_pad=n_pad)
    buf = C.c_void_p(1 << 20)
    for kind, P in (("qLogEI", 0), ("qEI", 31), ("EI", 0)):
        a = _lib.AcqSpec(kind=_lib.ACQ_KIND[kind], obj_scale=1.0)
        assert lib.bb_acq_grad_large(C.byref(m), C.byref(a), None, 0, P, buf, buf, buf, buf, buf, 1024, None, None,
                                     None) == 0
        assert lib.bb_acq_grad(C.byref(m), C.byref(a), None, 0, P, buf, buf, buf, buf, buf, 1024, None, None,
                               None) == _lib.BB_ERR_UNSUPPORTED


# ---- dispatch: engine.acq_grad_op ------------------------------------------------------------------------------------
@pytest.mark.parametrize("wide, n_pad, entry", [
    (False, 64, "acq_grad"),
    (False, 256, "acq_grad"),
    (False, 320, "acq_grad_large"),
    (False, 1024, "acq_grad_large"),
    (True, 128, "acq_grad_large"),
    (True, 1024, "acq_grad_large"),
])
def test_dispatch_picks_bb_acq_grad_for_small_models_and_the_large_entry_otherwise(wide, n_pad, entry):
    from baybe_b200 import _lib
    from baybe_b200.engine import acq_grad_op

    assert _lib.GRAD_MAX_NPAD == 256
    assert acq_grad_op(_fake(wide=wide, n_pad=n_pad)) is getattr(torch.ops.baybe_b200, entry)


def test_task_models_still_raise(lib):
    from baybe_b200 import _lib
    from baybe_b200.engine import acq_grad_op

    # the host path rejects them before any gradient call
    rng = np.random.default_rng(0)
    X = rng.uniform(0, 1, (12, 2))
    gp = OracleGradGP(X, np.sin(3 * X).sum(1), np.array([np.zeros(2), np.ones(2)]), "matern52", np.full(2, 0.4), 1e-3)
    gp.task_col = 1
    with pytest.raises(NotImplementedError, match="single-task"):
        recommend_continuous_hybrid(gp, AcqConfig("qEI"), np.zeros((1, 0)), np.array([[0.0, 0.0], [1.0, 1.0]]), 1)
    if torch.cuda.is_available():
        return
    # and both entry points reject them, whichever acq_grad_op picks
    buf = C.c_void_p(1 << 20)
    a = _lib.AcqSpec(kind=_lib.ACQ_KIND["qEI"], obj_scale=1.0)
    for wide, n_pad, entry in ((False, 64, "bb_acq_grad"), (False, 512, "bb_acq_grad_large"),
                               (True, 128, "bb_acq_grad_large")):
        m = _fake(wide=wide, task=True, n_pad=n_pad)
        assert acq_grad_op(m) is getattr(torch.ops.baybe_b200, entry[3:])
        rc = getattr(lib, entry)(C.byref(m), C.byref(a), buf, 10, 0, None, None, None, None, buf, 64, buf, buf, None)
        assert rc == _lib.BB_ERR_UNSUPPORTED
        assert lib.bb_last_error() == f"{entry}: models with a task parameter are not supported".encode()
