"""dynamic_factor_models_b200 -- H100-native hot path of QuantEcon/dynamic_factor_models.

Host-side mirror (Python; the Julia shim that a
maintainer would add is julia/DFMB200.jl, see INTEGRATION.md) of the reference's `dfm_functions`
surface over the C ABI in include/dfm_b200.h.  All arithmetic runs in hand-written sm_90a CUDA
kernels inside lib/libdfm_b200.so; there is no CPU fallback: importing works without a GPU, but
creating a handle raises if the library or a CUDA device is missing.
"""
from ._lib import Library, DFMError, default_library_path  # noqa: F401
from .api import (  # noqa: F401
    instability_tests, fitted_value_correlations,
    DFMModel, VARModel, FactorEstimateStats, NonParametric, Parametric, LambdaConstraint,
    construct_constraint, estimate, estimate_factor, estimate_factor_loading, estimate_var,
    impulse_response, bai_ng_criterion, amengual_watson_test, estimate_factor_numbers,
    standardize_data, pca_score, em_kalman, em_init_from_factors, set_default_library, get_library,
    kalman_smooth, forecast, posterior_draws, forecast_bands, news,
)
from . import ingest  # noqa: F401   (host-side panel ingestion: the step before the path)
