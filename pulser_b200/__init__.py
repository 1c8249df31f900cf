"""pulser_b200: H100-native (sm_90a) time-evolution emulator for Pulser sequences.

Public names mirror ``pulser_simulation/__init__.py`` (``QutipEmulator`` -> ``B200Emulator``, ``QutipBackendV2`` ->
``B200Backend``, ``QutipBackend`` -> ``B200LegacyBackend``, ``QutipConfig / QutipState / QutipOperator`` ->
``B200Config / B200State / B200Operator``, ``SimConfig`` -> the QuTiP-free ``SimConfig``); they resolve lazily so that the plain-array path (``engine``, ``spec``,
``workloads``) keeps working where pulser-core is not installed.
"""
from ._compat import HAVE_PULSER  # noqa: F401  (installs the import hooks)

__version__ = "0.1.0"

_LAZY = {
    "B200Emulator": ("emulator", "B200Emulator"),
    "Solver": ("emulator", "Solver"),
    "B200Backend": ("backend", "B200Backend"),
    "B200LegacyBackend": ("backend", "B200LegacyBackend"),
    "B200Config": ("backend", "B200Config"),
    "B200State": ("backend", "B200State"),
    "B200Operator": ("backend", "B200Operator"),
    "density_matrix_aggregator": ("backend", "density_matrix_aggregator"),
    "SimConfig": ("simconfig", "SimConfig"),
}

__all__ = ["HAVE_PULSER", *_LAZY]


def __getattr__(name: str):
    if name in _LAZY:
        import importlib

        module, attr = _LAZY[name]
        return getattr(importlib.import_module(f"{__name__}.{module}"), attr)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
