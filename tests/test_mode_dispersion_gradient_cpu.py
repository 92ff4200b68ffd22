"""CPU: the float64 model of the dispersion gradient (oracle/mode_dispersion_gradient.py) against dense eigen-decompositions of
the assembled operator, on the group-gradient CPU cases (which include a core with curved eps(f), where chi_1, chi_2 and p''
matter), and the binding side of ``"disp_eps"`` (b200ms_solve_batch_ext2) without a device.

For every case the core-summed d_g (d^2 lambda / df^2) must match the central difference of the exact second derivative of the
dense eigenpair (``mode_dispersion.second_derivatives``) under eps +- delta on the core, within twice the Richardson estimate of
that difference's step error; so must single PML, wall and bend sites (at fixed PML stretch).  The map must not depend on the free multiples of v in
x and x2 (with the matching multiple of x in x2), dropping x2 and w_hat2 must miss the bound by far, and
``plugin.dispersion_gradient_of`` must be the eps-difference limit of ``plugin.dispersion_of``."""
import ctypes as C
import re

import numpy as np
import pytest

from oracle import mode_dispersion as MD
from oracle import mode_dispersion_gradient as DG
from oracle import restatement as R
from tests.test_fourth_order_binding_cpu import HEADER, NoHandle, _header_fields, _problem
from tests.test_mode_derivatives_cpu import F0, _operator
from tests.test_mode_dispersion_cpu import CASES2, _setup
from tests.test_mode_group_gradient_cpu import COMPS, _fundamental, _pair_near
from tidy3d_b200 import _cabi, plugin
from tidy3d_b200.solver import compute_modes_batch

STEP = 1e-3 * 12.0  # eps step of the central differences (and half of it)


def _inputs(c):
    if not c["disp"]:
        return dict()
    return dict(eps_dfreq=c["deps_at"](F0), eps_d2freq=c["d2eps_at"](F0) if "d2eps_at" in c else None)


def _model(c, v, lam, **kw):
    return DG.dispersion_gradient(c["eps_at"](F0), (c["x"], c["y"]), F0, c["ms"], v, lam, c["sym"], c["mu"], **_inputs(c), **kw)


def _second(c, lam, comp, mask, d):
    """The dense eigenpair near lam under eps_comp + d on mask, and mode_dispersion.second_derivatives of it."""
    e = c["eps_at"](F0)
    e[comp] = e[comp] + d * mask
    lp, vp = _pair_near(_operator(c, F0, e), lam)
    return MD.second_derivatives(e, (c["x"], c["y"]), F0, c["ms"], vp, lp, c["sym"], c["mu"], **_inputs(c))


def _check(c, lam, out, comp, a, mask, floor=0.0):
    """d_g lambda'' summed over mask against the Richardson-bounded central difference; returns (|got - fd|, bound).  floor:
    the roundoff of lambda'' relative to itself, which the difference divides by the step (matters for single sites)."""
    def fd(d):
        return (_second(c, lam, comp, mask, d)["d2lam_dfreq2"] - _second(c, lam, comp, mask, -d)["d2lam_dfreq2"]) / (2 * d)

    f1, f2 = fd(STEP), fd(STEP / 2)
    got = np.sum(out["d2lam_dfreq2_deps"][a][mask])
    noise = floor * abs(_second(c, lam, comp, mask, 0.0)["d2lam_dfreq2"]) / STEP if floor else 0.0
    return abs(got - f2), 2 * abs(f1 - f2) / 3 + 1e-8 * abs(f2) + noise


@pytest.mark.parametrize("name", sorted(CASES2))
def test_core_sum_matches_dense_differences(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    out = _model(c, v, lam)
    for comp, a in COMPS:
        err, bound = _check(c, lam, out, comp, a, c["core"])
        print(f"[disp_eps] {name} row {a}: |d_g lambda'' - fd| {err:.2e}, bound {bound:.2e}")
        assert err <= bound, (a, err, bound)


@pytest.mark.parametrize("name, site", [("pml", (0, 6)), ("pml", (7, 11)), ("pmc_x_pec_y", (0, 6)), ("pmc_x_pec_y", (7, 0)),
                                        ("bend", (6, 5)), ("bend", (13, 6))])
def test_single_sites_match_dense_differences(name, site, monkeypatch):
    c = _setup(name)
    lam, v = _fundamental(c)
    out = _model(c, v, lam)
    # the map is taken at fixed PML stretch, and the PML speeds follow the mean eps of each strip: hold them at the unperturbed
    # values (the first call below) for the differences
    orig, held = R.pml_speeds, []

    def frozen(*args):
        if not held:
            held.append(orig(*args))
        return held[0]

    monkeypatch.setattr(R, "pml_speeds", frozen)
    _operator(c, F0)
    mask = np.zeros_like(c["core"])
    mask[site] = True
    for comp, a in COMPS:
        err, bound = _check(c, lam, out, comp, a, mask, floor=1e-13)
        assert err <= bound, (site, a, err, bound)


@pytest.mark.parametrize("name", ["plain", "pml", "all", "mu_diag", "dispersive_curved"])
def test_invariance_under_the_free_multiples(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    out = _model(c, v, lam)
    x, x2 = out["x"], out["x2"]
    ref = out["d2n_dfreq2_deps"]
    for alpha, beta in ((0.3 - 0.7j, 0.0), (2.0, -1.1 + 0.4j), (0.0, 0.5j)):
        moved = _model(c, v, lam, x=x + alpha * v, x2=x2 + alpha * x + beta * v)  # w_hat, w_hat2 formed from the moved x, x2
        assert np.abs(moved["d2n_dfreq2_deps"] - ref).max() <= 1e-12 * np.abs(ref).max(), (alpha, beta)


def test_second_order_corrections_are_needed():
    c = _setup("pml")
    lam, v = _fundamental(c)
    zero = np.zeros_like(v)
    out = _model(c, v, lam, x2=zero, w_hat2=zero)
    missed = []
    for comp, a in COMPS:
        err, bound = _check(c, lam, out, comp, a, c["core"])
        missed.append(err / bound)
    print(f"[disp_eps] pml without x2, w_hat2: |error| / bound {missed}")
    assert max(missed) > 10, missed


def test_dispersion_gradient_of_is_the_limit_of_differences_of_dispersion_of():
    c = _setup("dispersive_curved")
    lam, v = _fundamental(c)
    out = _model(c, v, lam)
    core = c["core"]
    got = plugin.dispersion_gradient_of(F0, out["d2n_dfreq_deps"], out["d2n_dfreq2_deps"])
    assert np.array_equal(got, out["dispersion_deps"])
    for comp, a in COMPS:
        def disp(d):
            s = _second(c, lam, comp, core, d)
            return plugin.dispersion_of(F0, s["dn_dfreq"], s["d2n_dfreq2"])

        fds = [(disp(d) - disp(-d)) / (2 * d) for d in (STEP, STEP / 2)]
        want = np.sum(got[a][core])
        bound = 2 * abs(fds[0] - fds[1]) / 3 + 1e-8 * abs(fds[1])
        assert abs(want - fds[1]) <= bound, (a, want, fds, bound)
        # the check is not vacuous (the x-polarised fundamental barely sees eps_yy: there the bound is some 10 % of the sum)
        assert bound <= (0.2 if a == 1 else 1e-3) * abs(want), (a, want, bound)


def test_pec_cells_report_zero():
    c = _setup("pml")
    eps = c["eps_at"](F0)
    for comp in (0, 4, 8):
        eps[comp] = eps[comp].copy()
        eps[comp][0, 5] = -1e8
    lam, v = _pair_near(_operator(c, F0, eps), _fundamental(c)[0])
    out = DG.dispersion_gradient(eps, (c["x"], c["y"]), F0, c["ms"], v, lam, c["sym"], c["mu"])
    assert (out["d2n_dfreq2_deps"][:, 0, 5] == 0).all() and np.abs(out["d2n_dfreq2_deps"]).max() > 0


def test_ext2_struct_mirrors_the_v212_header():
    assert _cabi.ABI_VERSION == 212
    assert [f for f, _ in _cabi.ResultExt2._fields_] == _header_fields("b200ms_result_ext2") == ["d2n_dfreq2_deps"]
    assert [f for f, _ in _cabi.ResultExt._fields_] == _header_fields("b200ms_result_ext") == ["d4n_dfreq4", "d4n_residual"]
    assert "b200ms_solve_batch_ext2" in _cabi.EXPORTS
    assert re.search(r"int b200ms_solve_batch_ext2\(b200ms_handle \*h, int nprob, const b200ms_problem \*prob, b200ms_result \*res,\s*"
                     r"const b200ms_problem_ext \*pext,\s*const b200ms_result_ext \*rext, const b200ms_result_ext2 \*rext2\);",
                     open(HEADER).read())


def test_disp_eps_is_checked_before_a_handle_is_taken():
    with pytest.raises(AssertionError, match="handle used"):  # a valid request gets as far as the handle
        compute_modes_batch([_problem()], handle=NoHandle(), derivatives=("disp_eps",))
    with pytest.raises(ValueError, match="unknown derivative"):
        compute_modes_batch([_problem()], handle=NoHandle(), derivatives=("disp_epsilon",))


def test_buffers_handed_to_the_library():
    # a handle without a device context: b200ms_solve_batch_ext2 rejects the null handle before any CUDA call
    h = _cabi.Handle.__new__(_cabi.Handle)
    h._h = C.c_void_p()
    p = _problem()
    pk = _cabi.PackedProblem(p["eps_cross"], p["coords"], p["freq"], p["mode_spec"], fourth=True)
    kw = dict(want_fields=False, want_dfreq=True, want_deps=True, want_d2freq=True, want_group_eps=True, want_d3freq=True, want_d4freq=True)
    rc, _, _, res = h.solve_batch([pk], want_d2freq2_deps=True, **kw)
    assert rc == _cabi.ERR_ARG
    assert h.last_d2n_dfreq2_deps[0].shape == (3, 16, 16, 2)
    assert res[0].d2n_dfreq_deps
    for drop in ("want_group_eps", "want_d4freq"):
        with pytest.raises(ValueError, match="want_d2freq2_deps"):
            h.solve_batch([pk], want_d2freq2_deps=True, **dict(kw, **{drop: False}))
