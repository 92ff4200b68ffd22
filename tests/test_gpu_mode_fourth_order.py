"""GPU: d^4 n / df^4 of the fourth-order pass (fourth_rhs_kernel, fourth_scan_kernel, csrc/derivatives.cuh) against the float64
model (oracle/mode_fourth_order.py) on the device's own eigenvectors, against device finite differences (also with a core whose
eps(f) is quartic), for eps_d4freq arrays against section tables, for bit-identical other outputs and batch invariance, for the
NaN rule of the two correction solves, and for the rejected scope."""
import dataclasses

import numpy as np
import pytest

from oracle import mode_fourth_order as M4
from tests.golden.cases import CASES as GOLDEN_CASES
from tests.test_gpu_mode_dispersion import CASES, F0, _problem, _strip
from tidy3d_b200 import plugin
from tidy3d_b200 import workloads as W
from tidy3d_b200.sections import Medium, Section
from tidy3d_b200.solver import TOLERANCES, compute_modes_batch, get_handle

pytestmark = pytest.mark.gpu
# device against the model on the device's own eigenvectors (tight preset): 10 x the largest relative error measured on an
# H100 80GB HBM3 at a 700 W power limit (1.27e-9, pml_96 and minus_96; the other cases 7.3e-11 to 1.1e-9), DESIGN.md §6
MODEL_RTOL = 1.3e-8
QUARTIC = (0.05, 0.2, 0.3, 3.0)  # eps(f) = eps0 (1 + a u + b u^2 + c u^3 + d u^4), u = f / F0 - 1
STEPS = (6e-2, 3e-2)


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_matches_model_on_its_own_eigenvectors(name):
    p = _problem(name)
    h = get_handle(tolerance="tight")
    (res,), (info,) = compute_modes_batch([p], handle=h, return_info=True, derivatives=("freq4",))
    fields, n = res[0], res[1]
    errs = []
    for m in range(p["mode_spec"].num_modes):
        v = np.r_[fields[0, 0, :, :, 0, m].ravel(), fields[0, 1, :, :, 0, m].ravel()]
        out = M4.fourth_derivatives(list(p["eps_cross"]), p["coords"], p["freq"], p["mode_spec"], v, -(n[m] ** 2), p["symmetry"])
        errs.append(abs(info["d4n_dfreq4"][m] - out["d4n_dfreq4"]) / abs(out["d4n_dfreq4"]))
        fq = p["freq"]
        assert np.isclose(info["beta4"][m], plugin.beta4_of(fq, info["d3n_dfreq3"][m], info["d4n_dfreq4"][m]), rtol=1e-14, atol=0)
    print(f"[fourth] {name}: max relative |d4n_dfreq4 - model| = {max(errs):.3e}, residuals {info['d4n_residual']}")
    assert max(errs) <= MODEL_RTOL, errs


def _fourth(n, s):
    """Scaled fourth central difference of n at F0 over the solves at F0 (1 - 2s, 1 - s, 1, 1 + s, 1 + 2s)."""
    return (n[4] - 4 * n[3] + 6 * n[2] - 4 * n[1] + n[0]).real / s**4


def _fd_check(make, hs=STEPS):
    """f^4 Re n'''' of the device's ("freq4",) pass at F0 against device solves at F0, F0 (1 +- h), F0 (1 +- 2h), Richardson
    extrapolated over the two steps.  Returns (analytic f^4 Re n'''', bound)."""
    h = get_handle(tolerance="tight")
    (_,), (info,) = compute_modes_batch([make(F0)], handle=h, want_fields=False, return_info=True, derivatives=("freq4",))
    g4 = []
    for s in hs:
        freqs = [F0 * (1 + k * s) for k in (-2, -1, 0, 1, 2)]
        g4.append(_fourth(np.array([r[1] for r in compute_modes_batch([make(f) for f in freqs], handle=h, want_fields=False)]), s))
    rich = (4 * g4[1] - g4[0]) / 3
    # the eigenvalue tolerance of the tight preset (n to a few 1e-9) enters a fourth difference as ~16 eig / h^4, and the
    # Richardson combination weighs the finer difference by 4/3
    eig = 4e-9
    bound = np.abs(g4[0] - g4[1]) + 22 * eig / hs[1] ** 4
    ana = F0**4 * info["d4n_dfreq4"].real
    print(f"[fourth] fd: analytic {ana}, richardson {rich}, bound {bound}")
    assert np.all(np.abs(ana - rich) <= bound), (ana, rich, bound)
    return ana, bound


@pytest.mark.parametrize("name", ["pml_96", "bend_lossy_64"])
def test_fourth_derivative_matches_device_finite_differences(name):
    p = _problem(name)
    _fd_check(lambda f: dict(p, freq=f))


def _quartic_medium(eps):
    core_eps = complex(eps[0].real.max())
    a, b, c, d = QUARTIC

    def e(f):
        u = f / F0 - 1
        return core_eps * (1 + a * u + b * u * u + c * u**3 + d * u**4)

    return core_eps, Medium(e)


def _quartic_section(eps):
    core_eps, core = _quartic_medium(eps)
    clad = Medium(complex(eps[0].real.min()))
    site = np.stack([np.isclose(eps[c].real, core_eps.real) for c in (0, 4, 8)]).astype(np.uint16)
    return Section(background=clad, media=[clad, core], site_medium=site)


def test_quartic_dispersive_section():
    eps, coords, ms = _strip(64)
    sec = _quartic_section(eps)
    ana, bound = _fd_check(lambda f: dict(section=sec, coords=coords, freq=f, mode_spec=ms))
    h = get_handle(tolerance="tight")
    (_,), (info_nd,) = compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms)], handle=h, want_fields=False,
                                           return_info=True, derivatives=("freq4",))
    print(f"[fourth] quartic section: f^4 n'''' {ana}, nondispersive {F0**4 * info_nd['d4n_dfreq4'].real}, bound {bound}")
    assert np.all(np.abs(ana - F0**4 * info_nd["d4n_dfreq4"].real) > 10 * bound)  # the material terms matter here


def test_eps_d4freq_input_matches_the_section():
    """The quartic core given as eps_cross arrays with eps_dfreq .. eps_d4freq agrees with the section's tables."""
    eps, coords, ms = _strip(64)
    core = eps[0].real > 5
    a, b, c, d = QUARTIC
    coef = (a / F0, 2 * b / F0**2, 6 * c / F0**3, 24 * d / F0**4)  # derivatives of the polynomial at u = 0
    arrs = [np.zeros_like(eps) for _ in range(4)]
    for k in (0, 4, 8):
        for arr, ck in zip(arrs, coef):
            arr[k] = np.where(core, eps[k] * ck, 0)
    sec = _quartic_section(eps)
    h = get_handle(tolerance="tight")
    (_,), (ia,) = compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms, eps_dfreq=arrs[0], eps_d2freq=arrs[1],
                                            eps_d3freq=arrs[2], eps_d4freq=arrs[3])],
                                      handle=h, want_fields=False, return_info=True, derivatives=("freq4",))
    (_,), (ib,) = compute_modes_batch([dict(section=sec, coords=coords, freq=F0, mode_spec=ms)], handle=h, want_fields=False,
                                      return_info=True, derivatives=("freq4",))
    # the section's tables are central differences of eps(f) (relative steps 1e-4, 1e-3, 1e-3 and 5e-3)
    err = np.abs(ia["d4n_dfreq4"] - ib["d4n_dfreq4"]).max() / np.abs(ia["d4n_dfreq4"]).max()
    print(f"[fourth] eps_d4freq against section tables: {err:.3e}")
    assert err <= 1e-4


def test_fourth_order_changes_nothing_else_and_does_not_depend_on_the_batch():
    wl = W.si_strip(64, 2, W.sweep_freqs(64))
    eps = np.ascontiguousarray(np.stack(wl.eps_cross))
    probs = [dict(eps_cross=eps, coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec) for f in wl.freqs]
    h = get_handle()
    base, i1 = compute_modes_batch(probs, handle=h, return_info=True, derivatives=("group_eps", "freq3"))
    fourth, i2 = compute_modes_batch(probs, handle=h, return_info=True, derivatives=("group_eps", "freq4"))
    keys = ("dn_dfreq", "dn_deps", "d2n_dfreq2", "d2n_residual", "dispersion", "d2n_dfreq_deps", "dng_deps", "d3n_dfreq3",
            "dispersion_slope", "beta3")
    for a, b, x, y in zip(base, fourth, i1, i2):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        for k in keys:
            assert np.array_equal(x[k], y[k], equal_nan=True), k
        assert np.all(np.isfinite(y["d4n_dfreq4"]))
    (alone,), (ia,) = compute_modes_batch([probs[17]], handle=h, return_info=True, derivatives=("freq4",))
    # one problem alone may stop at a different iterate of the eigen-solve and of its correction solves (within the tolerances)
    err = np.abs(ia["d4n_dfreq4"] - i2[17]["d4n_dfreq4"]).max() / np.abs(ia["d4n_dfreq4"]).max()
    print(f"[fourth] alone against batch position 17: {err:.3e}")
    assert err <= 1e-3


def test_near_degenerate_pml_pair_nan_rule():
    fac, _, _ = GOLDEN_CASES["pml_none_128"]
    wl = fac()
    h = get_handle()
    (_,), (info,) = compute_modes_batch([dict(eps_cross=wl.eps_cross, coords=wl.coords, freq=wl.freqs[0], mode_spec=wl.mode_spec)], handle=h,
                                        want_fields=False, return_info=True, derivatives=("freq4",))
    d4 = info["d4n_dfreq4"]
    tol = TOLERANCES["reference"]["inner_tol"]
    stopped = (info["d2n_residual"] > 100 * tol) | (info["d4n_residual"] > 100 * tol)
    print(f"[fourth] pml_none_128: d4n NaN {np.isnan(d4).tolist()}, residuals {info['d2n_residual']} / {info['d4n_residual']}")
    assert np.array_equal(np.isnan(d4), stopped)
    assert np.array_equal(np.isnan(info["beta4"]), stopped)


def test_scope():
    eps, coords, ms = _strip(48)
    h = get_handle()
    angled = dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=dataclasses.replace(ms, angle_theta=0.2))
    for left in (False, True):
        with pytest.raises(NotImplementedError):
            compute_modes_batch([angled], handle=h, derivatives=("freq4",), left_solve=left)
    basis = np.zeros((6, 48, 48, 1, ms.num_modes), complex)
    basis[0, 20:28, 20:28] = 1.0
    basis[1, 20:28, 20:28, 0, 1] = 1.0
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms, solver_basis_fields=basis)], handle=h, derivatives=("freq4",))
    pec = eps.copy()
    for c in (0, 4, 8):
        pec[c][:4] = -1e8
    mu = [np.ones((48, 48), complex) if k in (0, 4, 8) else np.zeros((48, 48), complex) for k in range(9)]
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=pec, coords=coords, freq=F0, mode_spec=ms, mu_cross=mu)], handle=h, derivatives=("freq4",))
