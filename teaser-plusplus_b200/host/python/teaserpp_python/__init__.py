"""`teaserpp_python` for the GPU-native path.

Public surface = the reference package's (python/teaserpp_python/__init__.py): the pybind11 classes re-exported from
`_teaserpp`, the v1.0 enum aliases on the solver / certifier classes, `RobustRegistrationSolverParams` (a named tuple
of the fourteen constructor arguments with the reference's defaults, in constructor order) and the `params` attribute
that hands back the positional arguments a solver object was built with.
"""
import collections
import functools

from . import _teaserpp as _ext

# ---- re-exports -----------------------------------------------------------------------------------------------------
_PUBLIC = ("OMP_MAX_THREADS", "CertificationResult", "DRSCertifier", "EigSolverType", "InlierGraphFormulation",
           "InlierSelectionMode", "RegistrationSolution", "RobustRegistrationSolver", "RotationEstimationAlgorithm")
globals().update({name: getattr(_ext, name) for name in _PUBLIC})

# ---- v1.0 spellings of the enums, kept as class attributes ----------------------------------------------------------
for _owner, _alias, _enum in ((_ext.RobustRegistrationSolver, "ROTATION_ESTIMATION_ALGORITHM", "RotationEstimationAlgorithm"),
                              (_ext.RobustRegistrationSolver, "INLIER_SELECTION_MODE", "InlierSelectionMode"),
                              (_ext.RobustRegistrationSolver, "INLIER_GRAPH_FORMULATION", "InlierGraphFormulation"),
                              (_ext.DRSCertifier, "EIG_SOLVER_TYPE", "EigSolverType")):
    setattr(_owner, _alias, getattr(_ext, _enum))

# ---- constructor arguments as a named tuple (field order = the 14-argument constructor, registration.h:524-539) -----
_CTOR_ARGS = collections.OrderedDict(
    noise_bound=0.01,
    cbar2=1,
    estimate_scaling=True,
    rotation_estimation_algorithm=_ext.RotationEstimationAlgorithm.GNC_TLS,
    rotation_gnc_factor=1.4,
    rotation_max_iterations=100,
    rotation_cost_threshold=1e-6,
    rotation_tim_graph=_ext.InlierGraphFormulation.CHAIN,
    inlier_selection_mode=_ext.InlierSelectionMode.PMC_EXACT,
    kcore_heuristic_threshold=0.5,
    use_max_clique=True,
    max_clique_exact_solution=True,
    max_clique_time_limit=3600,
    max_clique_num_threads=_ext.OMP_MAX_THREADS,
)
RobustRegistrationSolverParams = collections.namedtuple("RobustRegistrationSolverParams", list(_CTOR_ARGS),
                                                        defaults=list(_CTOR_ARGS.values()))


# ---- solver.params: whatever positional arguments the object was constructed with -----------------------------------
def _install_params_attribute(cls):
    ctor = cls.__init__

    @functools.wraps(ctor)
    def recording_ctor(obj, *positional, **named):
        ctor(obj, *positional, **named)
        obj._params = positional

    cls.__init__ = recording_ctor
    cls.params = property(lambda obj: obj._params)


_install_params_attribute(_ext.RobustRegistrationSolver)

__all__ = list(_PUBLIC) + ["RobustRegistrationSolverParams"]
