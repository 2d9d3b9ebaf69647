"""CPU-side checks of the product's C-ABI: the library loads, exports every symbol declared in
include/teaser_b200.h, reports the reference's Params defaults, and FAILS LOUDLY without a GPU
(no compute calls are made here)."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ensure_built():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()


def test_header_symbols_exported():
    _ensure_built()
    hdr = open(os.path.join(ROOT, "include", "teaser_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = set(re.findall(r"\b(tzr_[a-z0-9_]+)\s*\(", hdr))
    assert len(names) >= 20
    L = C.CDLL(capi.LIB_PATH)
    for nme in sorted(names):
        assert hasattr(L, nme), f"{nme} declared in include/teaser_b200.h but not exported"
    assert set(capi._SYMBOLS) == names


def test_max_clique_batch_signature():
    """tzr_max_clique_batch is an added symbol (the ABI version stays 2) with the argument order the binding uses."""
    _ensure_built()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "teaser_b200.h")).read(), flags=re.S)
    m = re.search(r"int\s+tzr_max_clique_batch\s*\(([^)]*)\)", hdr)
    assert m, "tzr_max_clique_batch missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == ["ctx", "B", "n", "adj_bits", "mode", "kcore_heuristic_threshold", "time_limit_s", "cliques",
                    "clique_sizes", "proven_optimal", "search_flags"]
    assert len(capi.lib().tzr_max_clique_batch.argtypes) == len(args)
    assert capi.lib().tzr_abi_version() == 2


def test_params_defaults_match_reference():
    _ensure_built()
    p = capi.default_params()
    # teaser/include/teaser/registration.h:419-514
    assert p.noise_bound == 0.01 and p.cbar2 == 1 and p.estimate_scaling == 1
    assert p.rotation_estimation_algorithm == 0 and p.rotation_gnc_factor == 1.4
    assert p.rotation_max_iterations == 100 and p.rotation_cost_threshold == 1e-6
    assert p.rotation_tim_graph == 0 and p.inlier_selection_mode == 0
    assert p.kcore_heuristic_threshold == 0.5 and p.use_max_clique == 1 and p.max_clique_exact_solution == 1
    assert p.max_clique_time_limit == 3600
    assert capi.lib().tzr_words_per_row(5000) == 79
    assert capi.lib().tzr_abi_version() == 2


def test_struct_layouts_agree():
    import oracle_lib as orc
    assert C.sizeof(capi.Params) == C.sizeof(orc.Params) == 88
    assert C.sizeof(capi.Solution) == C.sizeof(orc.Solution)
    for (a, _), (b, _) in zip(capi.Solution._fields_, orc.Solution._fields_):
        assert a == b and getattr(capi.Solution, a).offset == getattr(orc.Solution, b).offset


def test_no_cpu_fallback():
    _ensure_built()
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("GPU present")
    except ImportError:
        pass
    with pytest.raises(capi.TzrError):
        capi.Context(0)


def test_product_does_not_reference_oracle():
    pkg = os.path.join(ROOT, "teaser-plusplus_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".cu", ".cuh", ".h", ".hpp", ".cc", ".cpp", ".py")):
                txt = open(os.path.join(dp, f), errors="ignore").read()
                assert "oracle_lib" not in txt and "libteaser_oracle" not in txt and "teaser_oracle" not in txt, f
