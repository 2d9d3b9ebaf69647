"""CPU checks of the batched front end's C-ABI: both entry points are exported by the library, declared in the header
with the argument list the Python binding passes, and listed among the symbols capi.lib() checks."""
import importlib
import os
import re

import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

BATCH = {
    "tzr_compute_fpfh_batch": ["ctx", "B", "n", "pts", "normal_search_radius", "fpfh_search_radius", "fpfh_out",
                               "normals_out", "status"],
    "tzr_match_correspondences_batch": ["ctx", "B", "ns", "src_pts", "nd", "dst_pts", "src_feat", "dst_feat", "dim",
                                        "use_absolute_scale", "use_crosscheck", "use_tuple_test", "tuple_scale",
                                        "tuple_seeds", "pairs", "capacity", "n_pairs", "global_scale"],
}


@pytest.mark.parametrize("name", sorted(BATCH))
def test_batch_symbol_exported_declared_and_bound(name):
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "teaser_b200.h")).read(), flags=re.S)
    m = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)", hdr)
    assert m, f"{name} missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == BATCH[name]
    assert name in capi._SYMBOLS
    assert len(getattr(capi.lib(), name).argtypes) == len(args)
