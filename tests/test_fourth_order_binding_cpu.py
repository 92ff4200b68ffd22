"""CPU: the binding side of the fourth frequency derivative (b200ms_solve_batch_ext) -- the ext structs against the header, the
argument checks of ``"freq4"`` and ``eps_d4freq`` before any handle is taken, and the buffers the binding hands to the library
-- without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tidy3d_b200 import _cabi
from tidy3d_b200 import workloads as W
from tidy3d_b200.sections import Medium, Section
from tidy3d_b200.solver import compute_modes_batch

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200ms.h")


class NoHandle:  # taking it would be an error: the checks come first
    @property
    def lock(self):
        raise AssertionError("handle used")


def _problem(**kw):
    wl = W.si_strip(16, 2, W.sweep_freqs(16))
    return dict(eps_cross=np.ascontiguousarray(np.stack(wl.eps_cross)), coords=wl.coords, freq=float(wl.freqs[0]), mode_spec=wl.mode_spec,
                **kw)


def _header_fields(name):
    text = open(HEADER).read()
    body = text[: text.index("} " + name + ";")].rsplit("typedef struct {", 1)[1]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return re.findall(r"(\w+)\s*;", body)


def test_ext_structs_mirror_the_v212_header():
    assert _cabi.ABI_VERSION == 212
    assert [f for f, _ in _cabi.ProblemExt._fields_] == _header_fields("b200ms_problem_ext") == ["eps_d4freq", "d4eps_table"]
    assert [f for f, _ in _cabi.ResultExt._fields_] == _header_fields("b200ms_result_ext") == ["d4n_dfreq4", "d4n_residual"]
    # the existing structs are unchanged: the new inputs and outputs live only in the ext structs
    assert [f for f, _ in _cabi.Problem._fields_][-1] == "left_solve"
    assert [f for f, _ in _cabi.Result._fields_][-2:] == ["dn_deps_tensor", "left_paired"]
    assert "b200ms_solve_batch_ext" in _cabi.EXPORTS
    assert re.search(r"int b200ms_solve_batch_ext\(b200ms_handle \*h, int nprob, const b200ms_problem \*prob, b200ms_result \*res,\s*"
                     r"const b200ms_problem_ext \*pext,\s*const b200ms_result_ext \*rext\);", open(HEADER).read())


def test_freq4_and_eps_d4freq_are_checked_before_a_handle_is_taken():
    with pytest.raises(AssertionError, match="handle used"):  # a valid request gets as far as the handle
        compute_modes_batch([_problem()], handle=NoHandle(), derivatives=("freq4",))
    with pytest.raises(ValueError, match="unknown derivative"):
        compute_modes_batch([_problem()], handle=NoHandle(), derivatives=("freq5",))
    bad = [np.zeros((16, 15), complex)] * 9
    with pytest.raises(ValueError, match="eps_d4freq"):
        compute_modes_batch([_problem(eps_d4freq=bad)], handle=NoHandle(), derivatives=("freq4",))
    with pytest.raises(ValueError, match="eps_d4freq"):
        compute_modes_batch([_problem(eps_d4freq=[np.zeros((16, 16), complex)] * 3)], handle=NoHandle(), derivatives=("freq4",))
    p = _problem()
    sec = Section(background=Medium(2.0))
    with pytest.raises(ValueError, match="eps_d4freq"):
        _cabi.PackedProblem(None, p["coords"], p["freq"], p["mode_spec"], section=sec, eps_d4freq=[np.zeros((16, 16), complex)] * 9)


def test_section_tables_and_medium_step():
    core = Medium(lambda f: 12.0 * (1 + 0.3 * (f / 2e14 - 1) ** 4))
    clad = Medium(2.07)
    assert Section(background=clad).d4_table(2e14) is None  # no dispersive medium
    sec = Section(background=clad, media=[clad, core])
    t = sec.d4_table(2e14)
    assert t.shape == (2, 9) and np.all(t[0] == 0)
    want = 12.0 * 0.3 * 24 / 2e14**4  # a quartic eps(f): the fourth difference is exact up to roundoff
    assert np.allclose(t[1][[0, 4, 8]], want, rtol=1e-5, atol=0)
    assert np.all(t[1][[1, 2, 3, 5, 6, 7]] == 0)


def test_buffers_handed_to_the_library():
    # a handle without a device context: b200ms_solve_batch_ext rejects the null handle before any CUDA call
    h = _cabi.Handle.__new__(_cabi.Handle)
    h._h = C.c_void_p()
    p = _problem()
    d4 = [np.full((16, 16), 1e-50, complex)] * 9
    pk = _cabi.PackedProblem(p["eps_cross"], p["coords"], p["freq"], p["mode_spec"], eps_d4freq=d4, fourth=True)
    assert pk.ext.eps_d4freq and not pk.ext.d4eps_table
    rc, _, _, res = h.solve_batch([pk], want_fields=False, want_dfreq=True, want_d2freq=True, want_d3freq=True, want_d4freq=True)
    assert rc == _cabi.ERR_ARG
    assert h.last_d4n_dfreq4[0].shape == (2,) and h.last_d4n_residual[0].shape == (2,)
    assert res[0].d3n_dfreq3
    with pytest.raises(ValueError, match="want_d3freq"):
        h.solve_batch([pk], want_fields=False, want_d4freq=True)
