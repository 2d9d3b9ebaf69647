"""CPU checks of graph_strip2_kernel's strip order: strips_below and strip_decode, the functions the kernel runs, reached on
the host through tzr_graph_strip_schedule.  For every row-block count nt = 1 ... 512 (n up to 65536) and every strip
length L = 1 ... 15 that debug flag bits 28-31 can force, strip p = 0 ... strips_below(nt, L) - 1 must decode to the
p-th strip of the tiling in its documented order: row block I = 0 first, each row block's strips left to right, strip k
of row block I starting at column block I + k L.  So every (I, J0) of the tiling comes out exactly once, with
I <= J0 < nt and (J0 - I) mod L = 0, and the strips [J0, min(nt, J0 + L)) cover the upper triangle of 128-blocks once.
The decoder is a float square-root estimate with integer fix-up loops, so an off-by-one anywhere in the range shows here.
Over this range the estimate alone is already exact (emulated in FP32, it first misses at about 6.3 million strips,
far beyond the 131328 of nt = 512, L = 1), so the fix-up loops are a guard that this test cannot tell apart from no
guard: the test pins the decoder's output, not that redundancy."""
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "teaser_b200.h")

NT_MAX = 512   # 65536 correspondences, the largest problem the pipeline takes
L_MAX = 15     # the largest strip length the 4-bit flag field forces


@pytest.fixture(scope="module", autouse=True)
def _built():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()


def tiling(nt, L):
    """(I, J0) of every strip, in the documented order"""
    per_row = (nt - np.arange(nt) + L - 1) // L  # ceil((nt - I) / L) strips in row block I
    I = np.repeat(np.arange(nt), per_row)
    first = np.repeat(np.cumsum(per_row) - per_row, per_row)  # index of its row block's first strip
    return I, I + L * (np.arange(I.size) - first)


@pytest.mark.parametrize("L", range(1, L_MAX + 1))
def test_strip_decode_enumerates_the_tiling_once_in_order(L):
    for nt in range(1, NT_MAX + 1):
        I, J0 = capi.strip_schedule(nt, L)
        wI, wJ0 = tiling(nt, L)
        assert I.size == wI.size, f"nt={nt} L={L}: strips_below = {I.size}, the tiling has {wI.size} strips"
        assert np.all((I >= 0) & (I <= J0) & (J0 < nt)), f"nt={nt} L={L}: a strip outside I <= J0 < nt"
        assert np.all((J0 - I) % L == 0), f"nt={nt} L={L}: a strip not on its row block's L-grid"
        assert np.unique(I.astype(np.int64) * nt + J0).size == I.size, f"nt={nt} L={L}: a strip decoded twice"
        bad = np.flatnonzero((I != wI) | (J0 != wJ0))
        assert bad.size == 0, (f"nt={nt} L={L}: strip {bad[0]} decodes to ({I[bad[0]]}, {J0[bad[0]]}), "
                               f"the documented order has ({wI[bad[0]]}, {wJ0[bad[0]]})")
        # the blocks [J0, min(nt, J0 + L)) of all strips: the upper triangle of 128-blocks, each block once
        J = (J0[:, None] + np.arange(L)).ravel()
        Ik = np.repeat(I, L)
        keep = J < nt
        cover = np.bincount(Ik[keep].astype(np.int64) * nt + J[keep], minlength=nt * nt).reshape(nt, nt)
        assert np.array_equal(cover, np.triu(np.ones((nt, nt), dtype=np.int64))), f"nt={nt} L={L}: blocks not covered once"


def test_strip_schedule_refuses_out_of_range_arguments():
    lib = capi.lib()
    for nt, L in ((0, 4), (NT_MAX + 1, 4), (8, 0), (8, L_MAX + 1), (-1, 6)):
        assert lib.tzr_graph_strip_schedule(nt, L, None, None) == capi.TZR_ERR_INVALID_ARG, (nt, L)
    assert lib.tzr_graph_strip_schedule(NT_MAX, 1, None, None) == NT_MAX * (NT_MAX + 1) // 2


def test_strip_flag_field_bound_and_documented():
    assert capi.strip_flags(0) == 0 and capi.strip_flags(6) == 6 << 28 and capi.strip_flags(15) == 0xF0000000
    with pytest.raises(ValueError):
        capi.strip_flags(16)
    hdr = open(HEADER).read()
    assert "bits 28 to 31" in hdr
    code = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    for name, args in (("tzr_ctx_last_strip_blocks", ["ctx"]), ("tzr_graph_strip_schedule", ["nt", "L", "I", "J0"])):
        m = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)", code)
        assert m, f"{name} missing from the header"
        assert [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")] == args
        assert name in capi._SYMBOLS
        assert len(getattr(capi.lib(), name).argtypes) == len(args)
