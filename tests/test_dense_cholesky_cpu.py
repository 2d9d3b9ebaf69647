"""CPU checks of tzr_dense_cholesky_batch (the batched pose-graph routes' factorisation on given matrices): exported,
declared with its argument names and bound in capi; a call without a context refused with nothing written."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "tzr_dense_cholesky_batch"
ARGS = [("tzr_ctx*", "ctx"), ("int", "G"), ("const int32_t*", "n"), ("const double* const*", "A"),
        ("const double* const*", "b"), ("double* const*", "A_out"), ("double* const*", "x_out"), ("int32_t*", "info")]


@pytest.fixture(scope="module")
def header():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    return open(os.path.join(ROOT, "include", "teaser_b200.h")).read()


def test_symbol_exported_declared_and_bound(header):
    code = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    m = re.search(r"int\s+%s\s*\(([^)]*)\)" % NAME, code)
    assert m, f"{NAME} missing from the header"
    args = [a.strip() for a in " ".join(m.group(1).split()).split(",")]
    assert args == [f"{t} {nm}" for t, nm in ARGS]
    assert NAME in capi._SYMBOLS
    at = getattr(capi.lib(), NAME).argtypes
    dpp = C.POINTER(C.POINTER(C.c_double))
    assert at == [C.c_void_p, C.c_int, C.POINTER(C.c_int32), dpp, dpp, dpp, dpp, C.POINTER(C.c_int32)]
    assert callable(capi.Context.dense_cholesky_batch)


def raw_args(G=1, n=2):
    """The argument list of a G-matrix call (every matrix n x n) and the arrays behind it."""
    dp = C.POINTER(C.c_double)
    ns = np.full(max(1, G), n, dtype=np.int32)
    A = [np.eye(max(n, 1)) for _ in range(max(1, G))]
    b = [np.ones(max(n, 1)) for _ in range(max(1, G))]
    Ao = [np.full((max(n, 1), max(n, 1)), 7.0) for _ in range(max(1, G))]
    xo = [np.full(max(n, 1), 7.0) for _ in range(max(1, G))]
    info = np.full(max(1, G), 9, dtype=np.int32)
    ptrs = lambda arrs: (dp * len(arrs))(*[a.ctypes.data_as(dp) for a in arrs])
    args = [None, G, ns.ctypes.data_as(C.POINTER(C.c_int32)), ptrs(A), ptrs(b), ptrs(Ao), ptrs(xo),
            info.ctypes.data_as(C.POINTER(C.c_int32))]
    return args, (ns, A, b, Ao, xo, info)


def test_null_context_refused():
    L = capi.lib()
    args, keep = raw_args()
    assert getattr(L, NAME)(*args) == capi.TZR_ERR_INVALID_ARG
    _, _, _, Ao, xo, info = keep
    assert info[0] == 9 and (Ao[0] == 7.0).all() and (xo[0] == 7.0).all()  # nothing written
    for G in (0, -1):  # refused before the context is looked at
        args, keep = raw_args(G)
        assert getattr(L, NAME)(*args) == capi.TZR_ERR_INVALID_ARG
        assert keep[5][0] == 9
