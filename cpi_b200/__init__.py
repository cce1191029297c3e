"""cpi_b200 -- batched closed-form IMU preintegration (rpng/cpi hot path) on H100.

Everything computes in ``libcpi_b200.so`` (CUDA, sm_90a; C ABI in ``include/cpi_b200.h``); there is no CPU fallback.
Submodules are imported lazily so that ``import cpi_b200`` works on a box without the built extension:

    cpi_b200.capi      ctypes binding of the C ABI (``load()`` raises if the library is missing)
    cpi_b200.preint    CpiV1 / CpiV2 (reference-shaped), preintegrate(), preintegrate_host()
    cpi_b200.factor    ImuFactorCPIv1 / ImuFactorCPIv2 / JPLNavState, factor_eval(), factor_hessian(), predict_state(), retract()
    cpi_b200.shard     window sharding over ranks + one all-gather of the records
    cpi_b200.synth     seeded synthetic windows, .dat parser and the window builder replaying the reference driver loop
"""
__all__ = ["capi", "preint", "factor", "shard", "synth"]
__version__ = "0.1"


def __getattr__(name):
    if name in __all__:
        import importlib
        return importlib.import_module(f"{__name__}.{name}")
    raise AttributeError(name)
