"""CPU tests of ``bb_objective_grad_large``: its argument checks before any CUDA call, and the choice between it and
``bb_objective_grad`` (``engine.objective_grad_op``) on model structs filled by hand, which ``objectives._objective_grad``
follows."""
from __future__ import annotations

import ctypes as C

import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from baybe_b200 import _lib
    from baybe_b200.build import build

    build(verbose=False)
    return _lib.load()


def _fake(wide=False, task=False, n_pad=64, d=20):
    from tests.test_abi import _fake_model

    m = _fake_model(False, 1)
    m.n = m.n_pad = n_pad
    m.d = m.d_pad = d
    m.wide = int(wide)
    m.d_wide = d if wide else 0
    if task:
        m.task_col = 0
    return m


_BAD = [
    ("null models", "invalid", b"model array is null"),
    ("M = 0", "unsupported", b"n_targets=0"),
    ("M = 9", "unsupported", b"n_targets=9"),
    ("null spec", "invalid", b"acquisition spec is null"),
    ("null objective", "invalid", b"objective is null"),
    ("count mismatch", "invalid", b"objective of 1 targets for 2 models"),
    ("null model entry", "invalid", b"model 1 missing"),
    ("abi mismatch", "invalid", b"model 1 missing or ABI mismatch"),
    ("task", "unsupported", b"model 1: models with a task parameter are not supported"),
    ("n_pad 1088", "unsupported", b"n_pad=1088"),
    ("mixed d", "invalid", b"differs from model 0"),
    ("mixed family", "invalid", b"differs from model 0"),
    ("bad program", "invalid", b"unknown opcode"),
    ("kind 11", "invalid", b"not a single-objective"),
    ("negative N", "invalid", b"negative point count"),
    ("32 pending", "invalid", b"n_pending=32"),
    ("analytic with pending", "invalid", b"analytic kinds take no pending points"),
    ("S 0", "invalid", b"S=0"),
    ("S 1025", "invalid", b"S=1025"),
    ("null samples", "invalid", b"null base samples"),
    ("null pending", "invalid", b"pending points need"),
    ("null beta entry", "invalid", b"pending points need"),
    ("null output", "invalid", b"null buffer"),
]


def _grad_call(lib, case: str, N: int = 10, models=None):
    """bb_objective_grad_large on two hand-filled models (n_pad 512 and 64 unless `models` is given), qLogEI over a
    GEOM_MEAN of two bell programs, with `case` breaking one argument."""
    from baybe_b200 import _lib
    from baybe_b200.engine import objective_struct

    M = {"M = 0": 0, "M = 9": 9}.get(case, 2 if models is None else len(models))
    if models is None:
        models = [_fake(task=case == "task" and m == 1, n_pad=(1088 if case == "n_pad 1088" else 512) if m == 0 else 64)
                  for m in range(max(M, 1))]
    ms = models
    if case == "mixed d":
        ms[1].d += 1
    if case == "mixed family":
        ms[1].family = _lib.KERNEL_FAMILY["matern52"]
    if case == "abi mismatch":
        ms[1].abi_version = _lib.ABI_VERSION + 1
    arr = (C.POINTER(_lib.Model) * len(ms))(*(C.pointer(m) for m in ms))
    if case == "null model entry":
        arr[1] = C.POINTER(_lib.Model)()
    kind = {"kind 11": 11, "analytic with pending": _lib.ACQ_KIND["EI"]}.get(case, _lib.ACQ_KIND["qLogEI"])
    a = _lib.AcqSpec(kind=kind, obj_scale=1.0, tau_relu=1e-6, tau_max=1e-2, tau_pi=1e-3)
    Mo = min(max(M, 1), 8)
    if kind == _lib.ACQ_KIND["EI"]:
        progs, scal = [[(_lib.OBJ_OP["AFFINE"], (2.0, 1.0, 0.0))]] * Mo, 1 if Mo > 1 else 0
    else:
        progs, scal = [[(_lib.OBJ_OP["BELL"], (0.0, 1.0, 0.0))]] * Mo, 2 if Mo > 1 else 0
    obj = objective_struct(Mo, scal, progs, [1.0 / Mo] * Mo)
    obj.n_targets = 1 if case == "count mismatch" else M
    if case == "bad program":
        obj.prog[1][0].op = 99
    buf = C.c_void_p(1 << 20)
    P = {"analytic with pending": 1, "32 pending": 32, "null pending": 2, "null beta entry": 2}.get(case, 0)
    betas = (C.c_void_p * max(M, 1))(*([1 << 20] * max(M, 1)))
    if case == "null beta entry":
        betas[1] = None
    pend = None if case == "null pending" else buf
    S = {"S 0": 0, "S 1025": 1025}.get(case, 64)
    z = None if case == "null samples" else buf
    out = None if case == "null output" else buf
    N = -1 if case == "negative N" else N
    return lib.bb_objective_grad_large(None if case == "null models" else arr, M,
                                       None if case == "null spec" else C.byref(a),
                                       None if case == "null objective" else C.byref(obj), buf, N, P, pend, betas, pend,
                                       pend, pend, z, S, out, out, None)


@pytest.mark.parametrize("case, status, msg", _BAD, ids=[c for c, *_ in _BAD])
def test_objective_grad_large_rejects_bad_arguments_before_any_cuda_call(lib, case, status, msg):
    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    rc = _grad_call(lib, case)
    assert rc == {"invalid": _lib.BB_ERR_INVALID, "unsupported": _lib.BB_ERR_UNSUPPORTED}[status]
    assert msg in lib.bb_last_error()
    assert lib.bb_last_error().startswith(b"bb_objective_grad_large: ")


@pytest.mark.parametrize("shapes", [
    ((512, False), (64, False)),
    ((1024, False),) * 8,
    ((288, False),),
    ((256, True), (256, False)),
    ((200, False), (704, False)),
    ((1024, True), (128, False), (1024, False)),
], ids=["n512+n64", "M8-n1024", "n288", "wide+small", "n200+n704", "wide-n1024-mix"])
def test_objective_grad_large_takes_the_models_bb_objective_grad_rejects(lib, shapes):
    """Wide models, n_pad up to 1024 and mixes of them with small models pass every check of bb_objective_grad_large
    (N = 0 returns BB_OK before any CUDA call, with null buffers), where bb_objective_grad returns
    BB_ERR_UNSUPPORTED."""
    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    models = [_fake(wide=w, n_pad=n) for n, w in shapes]
    assert _grad_call(lib, "none", N=0, models=models) == 0
    M = len(models)
    arr = (C.POINTER(_lib.Model) * M)(*(C.pointer(m) for m in models))
    from baybe_b200.engine import objective_struct

    obj = objective_struct(M, 2 if M > 1 else 0, [[(_lib.OBJ_OP["BELL"], (0.0, 1.0, 0.0))]] * M, [1.0 / M] * M)
    a = _lib.AcqSpec(kind=_lib.ACQ_KIND["qLogEI"], obj_scale=1.0, tau_relu=1e-6, tau_max=1e-2, tau_pi=1e-3)
    buf = C.c_void_p(1 << 20)
    rc = lib.bb_objective_grad(arr, M, C.byref(a), C.byref(obj), buf, 10, 0, None, None, None, None, None, buf, 64,
                               buf, buf, None)
    assert rc == _lib.BB_ERR_UNSUPPORTED


def test_objective_grad_large_accepts_an_empty_point_set_with_null_buffers(lib):
    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    ms = [_fake(n_pad=512), _fake(n_pad=64)]
    arr = (C.POINTER(_lib.Model) * 2)(*(C.pointer(m) for m in ms))
    from baybe_b200.engine import objective_struct

    obj = objective_struct(2, 2, [[(_lib.OBJ_OP["BELL"], (0.0, 1.0, 0.0))]] * 2, [0.5, 0.5])
    a = _lib.AcqSpec(kind=_lib.ACQ_KIND["qLogEI"], obj_scale=1.0, tau_relu=1e-6, tau_max=1e-2, tau_pi=1e-3)
    buf = C.c_void_p(1 << 20)
    assert lib.bb_objective_grad_large(arr, 2, C.byref(a), C.byref(obj), None, 0, 0, None, None, None, None, None, buf,
                                       64, None, None, None) == 0


# ---- dispatch: engine.objective_grad_op ------------------------------------------------------------------------------
@pytest.mark.parametrize("shapes, entry", [
    (((64, False),), "objective_grad"),
    (((256, False), (64, False), (128, False)), "objective_grad"),
    (((288, False),), "objective_grad_large"),
    (((64, False), (288, False)), "objective_grad_large"),
    (((128, True),), "objective_grad_large"),
    (((64, False), (128, True)), "objective_grad_large"),
    (((224, False), (704, False)), "objective_grad_large"),
    (((1024, False),) * 8, "objective_grad_large"),
], ids=["small", "small-M3", "n288", "mixed-n288", "wide", "mixed-wide", "n224+n704", "M8-n1024"])
def test_dispatch_picks_bb_objective_grad_for_small_models_and_the_large_entry_otherwise(shapes, entry):
    from baybe_b200 import _lib
    from baybe_b200.engine import objective_grad_op

    assert _lib.GRAD_MAX_NPAD == 256
    assert objective_grad_op([_fake(wide=w, n_pad=n) for n, w in shapes]) is getattr(torch.ops.baybe_b200, entry)


def test_both_entries_reject_task_models(lib):
    from baybe_b200 import _lib
    from baybe_b200.engine import objective_grad_op, objective_struct

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    buf = C.c_void_p(1 << 20)
    a = _lib.AcqSpec(kind=_lib.ACQ_KIND["qLogEI"], obj_scale=1.0, tau_relu=1e-6, tau_max=1e-2, tau_pi=1e-3)
    obj = objective_struct(2, 2, [[(_lib.OBJ_OP["BELL"], (0.0, 1.0, 0.0))]] * 2, [0.5, 0.5])
    for shapes, entry in ((((64, False), (64, False)), "bb_objective_grad"),
                          (((64, False), (512, False)), "bb_objective_grad_large"),
                          (((64, False), (128, True)), "bb_objective_grad_large")):
        ms = [_fake(wide=w, n_pad=n, task=m == 1) for m, (n, w) in enumerate(shapes)]
        assert objective_grad_op(ms) is getattr(torch.ops.baybe_b200, entry[3:])
        arr = (C.POINTER(_lib.Model) * 2)(*(C.pointer(m) for m in ms))
        rc = getattr(lib, entry)(arr, 2, C.byref(a), C.byref(obj), buf, 10, 0, None, None, None, None, None, buf, 64,
                                 buf, buf, None)
        assert rc == _lib.BB_ERR_UNSUPPORTED
        assert lib.bb_last_error() == f"{entry}: model 1: models with a task parameter are not supported".encode()


# ---- the seam follows objective_grad_op -----------------------------------------------------------------------------
class _GP:
    def __init__(self, handle, n_pad, wide=False):
        self.handle = handle
        self.model = _fake(wide=wide, n_pad=n_pad)


@pytest.mark.parametrize("shapes, entry", [
    (((64, False), (128, False)), "objective_grad"),
    (((64, False), (320, False)), "objective_grad_large"),
    (((128, True),), "objective_grad_large"),
])
def test_objective_grad_seam_calls_the_op_objective_grad_op_picks(monkeypatch, shapes, entry):
    from baybe_b200 import objectives as ob
    from baybe_b200.engine import objective_grad_op

    picked, calls = [], []

    def spy(models):
        op = objective_grad_op(models)
        picked.append(op)
        return lambda *a: calls.append(a) or ("value", "grad")

    monkeypatch.setattr(ob, "objective_grad_op", spy)
    gps = [_GP(7 + m, n, w) for m, (n, w) in enumerate(shapes)]
    x = torch.zeros(3, 20)
    assert ob._objective_grad(gps, x, None, [], None, None, None, None, 0, [], 0, [], [], [], []) == ("value", "grad")
    assert picked == [getattr(torch.ops.baybe_b200, entry)]
    assert calls[0][0] is x and calls[0][1] == [gp.handle for gp in gps]
