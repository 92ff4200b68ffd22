"""tidy3d_b200 -- H100-native drop-in for the hot path of tidy3d's local mode solver.

Public surface (mirrors ``tidy3d.plugins.mode.solver``):
    compute_modes(eps_cross, coords, freq, mode_spec, ...) -> (fields, n_complex, eps_spec)
    compute_modes_batch([...])                              -> batched, one device call
"""
from .solver import compute_modes, compute_modes_batch  # noqa: F401

__all__ = ["compute_modes", "compute_modes_batch"]
