"""optuna_b200 -- GPU-native (H100, sm_90a) TPE suggestion engine (drop-in for optuna.samplers.TPESampler).

Host Python (this package) mirrors the reference's sampler plugin interface
(optuna/samplers/_base.py:31-228, optuna/samplers/_tpe/sampler.py:72) and calls hand-written
sm_90a CUDA through a C ABI (include/optuna_b200_tpe.h) bound with ctypes.
"""
from .engine import ParamSpec, TPEEngine  # noqa: F401

__all__ = ["ParamSpec", "TPEEngine", "B200TPESampler", "hypervolume_history", "plot_hypervolume_history",
           "best_trials", "pareto_front_info", "plot_pareto_front", "FanovaImportanceEvaluator",
           "RegretBoundEvaluator", "EMMREvaluator", "GPSampler", "terminator_improvement_history",
           "plot_terminator_improvement"]


def __getattr__(name):
    if name == "B200TPESampler":
        from .sampler import B200TPESampler
        return B200TPESampler
    if name in ("hypervolume_history", "plot_hypervolume_history", "best_trials", "pareto_front_info",
                "plot_pareto_front"):
        from . import analysis
        return getattr(analysis, name)
    if name == "FanovaImportanceEvaluator":
        from .importance import FanovaImportanceEvaluator
        return FanovaImportanceEvaluator
    if name in ("RegretBoundEvaluator", "EMMREvaluator", "terminator_improvement_history"):
        from . import terminator
        return getattr(terminator, name)
    if name == "plot_terminator_improvement":
        from .analysis import plot_terminator_improvement
        return plot_terminator_improvement
    if name == "GPSampler":
        from .gp_sampler import GPSampler
        return GPSampler
    raise AttributeError(name)
