"""CPU: the binding side of tensorial mode derivatives (left_solve, ABI v211) -- argument checks before any handle is taken, the
new struct fields, and the buffers the binding hands to the library -- without a device."""
import ctypes as C

import numpy as np
import pytest

from tidy3d_b200 import _cabi
from tidy3d_b200 import workloads as W
from tidy3d_b200.solver import compute_modes_batch


def _problem():
    wl = W.angled(16, num_modes=2)
    return dict(eps_cross=np.ascontiguousarray(np.stack(wl.eps_cross)), coords=wl.coords, freq=float(wl.freqs[0]), mode_spec=wl.mode_spec)


def test_left_solve_without_derivatives_is_an_argument_error():
    class NoHandle:  # taking it would be an error: the check comes first
        @property
        def lock(self):
            raise AssertionError("handle used")

    with pytest.raises(ValueError, match="left_solve"):
        compute_modes_batch([_problem()], handle=NoHandle(), left_solve=True)


def test_struct_fields_of_the_v212_header():
    assert _cabi.ABI_VERSION == 212
    assert [f for f, _ in _cabi.Problem._fields_][-1] == "left_solve"
    assert [f for f, _ in _cabi.Result._fields_][-2:] == ["dn_deps_tensor", "left_paired"]
    p = _problem()
    assert _cabi.PackedProblem(p["eps_cross"], p["coords"], p["freq"], p["mode_spec"], left_solve=True).struct.left_solve == 1
    assert _cabi.PackedProblem(p["eps_cross"], p["coords"], p["freq"], p["mode_spec"]).struct.left_solve == 0


def test_buffers_handed_to_the_library():
    # a handle without a device context: b200ms_solve_batch rejects the null handle before any CUDA call
    h = _cabi.Handle.__new__(_cabi.Handle)
    h._h = C.c_void_p()
    p = _problem()
    pk = _cabi.PackedProblem(p["eps_cross"], p["coords"], p["freq"], p["mode_spec"], left_solve=True)
    rc, _, _, res = h.solve_batch([pk], want_fields=False, want_dfreq=True, want_deps_tensor=True)
    assert rc == _cabi.ERR_ARG
    assert h.last_dn_deps[0].shape == (9, 16, 16, 2) and h.last_dn_dfreq[0].shape == (2,)
    assert not res[0].dn_deps and res[0].dn_deps_tensor
    with pytest.raises(ValueError):
        h.solve_batch([pk], want_fields=False, want_deps=True, want_deps_tensor=True)
