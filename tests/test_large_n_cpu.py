"""CPU checks of the size-limit and clique-route C-ABI: both entry points are exported by the library, declared in the
header with the argument list the Python binding passes, and listed among the symbols capi.lib() checks; the header
documents the two debug flags of the large clique route."""
import importlib
import os
import re

import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "teaser_b200.h")

SYMBOLS = {
    "tzr_ctx_set_max_n": ["ctx", "max_n"],
    "tzr_ctx_clique_route": ["ctx", "per_problem"],
}


@pytest.mark.parametrize("name", sorted(SYMBOLS))
def test_symbol_exported_declared_and_bound(name):
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    hdr = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)", hdr)
    assert m, f"{name} missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == SYMBOLS[name]
    assert name in capi._SYMBOLS
    assert len(getattr(capi.lib(), name).argtypes) == len(args)


def test_large_route_flags_documented():
    hdr = open(HEADER).read()
    assert "bit 19 (524288)" in hdr and "bit 20 (1048576)" in hdr
    assert "int tzr_ctx_set_max_n(" in hdr and "TZR_ABI_VERSION 2" in hdr
