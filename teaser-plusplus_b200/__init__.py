"""GPU-native TEASER++ registration hot path (package directory `teaser-plusplus_b200`).

Import with `importlib.import_module("teaser-plusplus_b200")` (the hyphen is part of the
contractual directory name).  Sub-modules:
  capi   — ctypes binding of the C-ABI shared library (csrc/libteaser_b200.so)
  synth  — synthetic workload generators for the BASELINE.json configs
"""
