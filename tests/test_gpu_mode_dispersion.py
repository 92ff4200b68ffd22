"""GPU: d^2 n / df^2 and the dispersion of the dispersion pass (csrc/derivatives.cuh) against the float64 model
(oracle/mode_dispersion.py) on the device's own eigenvectors, against device finite differences (also with a dispersive
core), for batch invariance, on a near-degenerate PML pair, and for the rejected scope."""
import dataclasses

import numpy as np
import pytest

from oracle import mode_dispersion as MD
from tests.golden.cases import CASES as GOLDEN_CASES
from tidy3d_b200 import plugin
from tidy3d_b200 import workloads as W
from tidy3d_b200.sections import Medium, Section
from tidy3d_b200.solver import TOLERANCES, compute_modes_batch, get_handle

pytestmark = pytest.mark.gpu
F0 = W.C_0 / 1.55
# device against the model on the device's own eigenvectors (tight preset): 10 x the largest relative error measured on an
# H100 80GB HBM3 (1.02e-9, pml_96 and minus_96), DESIGN.md §6
MODEL_RTOL = 1.1e-8


def _strip(n=64, **spec):
    wl = W.si_strip(n, 2)
    ms = dataclasses.replace(wl.mode_spec, **spec)
    return np.ascontiguousarray(np.stack(wl.eps_cross)), wl.coords, ms


def _lossy(eps):
    out = eps.copy()
    for c in (0, 4, 8):
        out[c] = np.where(out[c].real > 5, out[c] + 0.05j, out[c])
    return out


CASES = {
    "plain_64": dict(n=64),
    "pml_96": dict(n=96, spec=dict(num_pml=(10, 10))),
    "pmc_pec_64": dict(n=64, sym=(1, -1), spec=dict(num_pml=(0, 8))),
    "bend_lossy_64": dict(n=64, lossy=True, spec=dict(num_pml=(8, 8), bend_radius=6.0, bend_axis=1)),
    "minus_96": dict(n=96, direction="-", spec=dict(num_pml=(10, 10))),
}


def _problem(name):
    c = CASES[name]
    eps, coords, ms = _strip(c["n"], **c.get("spec", {}))
    if c.get("lossy"):
        eps = _lossy(eps)
    return dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=dataclasses.replace(ms, precision="double"),
                symmetry=c.get("sym", (0, 0)), direction=c.get("direction", "+"))


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_matches_model_on_its_own_eigenvectors(name):
    p = _problem(name)
    h = get_handle(tolerance="tight")
    (res,), (info,) = compute_modes_batch([p], handle=h, return_info=True, derivatives=("freq2",))
    fields, n = res[0], res[1]
    tol = TOLERANCES["tight"]["inner_tol"]
    errs = []
    for m in range(p["mode_spec"].num_modes):
        v = np.r_[fields[0, 0, :, :, 0, m].ravel(), fields[0, 1, :, :, 0, m].ravel()]
        out = MD.second_derivatives(list(p["eps_cross"]), p["coords"], p["freq"], p["mode_spec"], v, -(n[m] ** 2), p["symmetry"])
        assert info["d2n_residual"][m] <= 1.25 * tol, (m, info["d2n_residual"][m])
        err = abs(info["d2n_dfreq2"][m] - out["d2n_dfreq2"]) / abs(out["d2n_dfreq2"])
        errs.append(err)
        assert np.isclose(info["dispersion"][m], plugin.dispersion_of(F0, info["dn_dfreq"][m], info["d2n_dfreq2"][m]), rtol=1e-14, atol=0)
    print(f"[dispersion] {name}: max relative |d2n_dfreq2 - model| = {max(errs):.3e}")
    assert max(errs) <= MODEL_RTOL, errs


def _fd_check(make, h=None, hs=(1e-2, 5e-3)):
    """f^2 n'' and the dispersion of the device's ("freq2",) pass at F0 against device solves at F0 (1 -/+ step), Richardson
    extrapolated over the two steps.  Returns (analytic f^2 n'', bound)."""
    h = h or get_handle(tolerance="tight")
    (_,), (info,) = compute_modes_batch([make(F0)], handle=h, want_fields=False, return_info=True, derivatives=("freq2",))
    g2, dd = [], []
    for step in hs:
        freqs = [F0 * (1 - step), F0, F0 * (1 + step)]
        n3 = np.array([r[1] for r in compute_modes_batch([make(f) for f in freqs], handle=h, want_fields=False)])
        g2.append((n3[2] - 2 * n3[1] + n3[0]).real / step**2)  # f^2 Re n'' + O(step^2)
        dd.append(plugin.group_index(n3, freqs, step)[3][0])
    rich = (4 * g2[1] - g2[0]) / 3
    # the eigenvalue tolerance of the tight preset (n to a few 1e-9) enters a second difference as ~4 eig / step^2
    eig = 4e-9
    bound = np.abs(g2[0] - g2[1]) + 4 * eig / hs[1] ** 2
    ana = F0**2 * info["d2n_dfreq2"].real
    assert np.all(np.abs(ana - rich) <= bound), (ana, rich, bound)
    # the dispersion against plugin.group_index on the same solves (also Richardson extrapolated); D = -1e18 f (2 f n' + f^2 n'') / c0^2
    d_rich = (4 * dd[1] - dd[0]) / 3
    k = 1e18 * F0 / plugin.C0_UM**2
    d_bound = np.abs(dd[0] - dd[1]) + k * (4 * eig / hs[1] + 4 * eig / hs[1] ** 2)
    assert np.all(np.abs(info["dispersion"] - d_rich) <= d_bound), (info["dispersion"], d_rich, d_bound)
    return ana, bound


@pytest.mark.parametrize("name", ["pml_96", "bend_lossy_64"])
def test_second_derivative_matches_device_finite_differences(name):
    p = _problem(name)
    _fd_check(lambda f: dict(p, freq=f))


def test_dispersive_section():
    eps, coords, ms = _strip(64)
    core_eps = complex(eps[0].real.max())
    clad = Medium(complex(eps[0].real.min()))
    core = Medium(lambda f: core_eps * (1 + 0.05 * (f / F0 - 1) + 0.2 * (f / F0 - 1) ** 2))
    site = np.stack([np.isclose(eps[c].real, core_eps.real) for c in (0, 4, 8)]).astype(np.uint16)
    sec = Section(background=clad, media=[clad, core], site_medium=site)
    ana, bound = _fd_check(lambda f: dict(section=sec, coords=coords, freq=f, mode_spec=ms))
    h = get_handle(tolerance="tight")
    (_,), (info_nd,) = compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms)], handle=h, want_fields=False,
                                           return_info=True, derivatives=("freq2",))
    assert np.all(np.abs(ana - F0**2 * info_nd["d2n_dfreq2"].real) > 20 * bound)  # the material terms matter here


def test_eps_d2freq_input_matches_the_section():
    """The same dispersive core given as eps_cross arrays with eps_dfreq / eps_d2freq agrees with the section's tables."""
    eps, coords, ms = _strip(64)
    core = eps[0].real > 5
    a1, a2 = 0.05 / F0, 2 * 0.2 / F0**2  # d/df and d^2/df^2 of eps0 (1 + 0.05 u + 0.2 u^2) at u = 0, per unit eps0
    de, d2e = np.zeros_like(eps), np.zeros_like(eps)
    for c in (0, 4, 8):
        de[c] = np.where(core, eps[c] * a1, 0)
        d2e[c] = np.where(core, eps[c] * a2, 0)
    core_eps = complex(eps[0].real.max())
    med = Medium(lambda f: core_eps * (1 + 0.05 * (f / F0 - 1) + 0.2 * (f / F0 - 1) ** 2))
    clad = Medium(complex(eps[0].real.min()))
    site = np.stack([np.isclose(eps[c].real, core_eps.real) for c in (0, 4, 8)]).astype(np.uint16)
    sec = Section(background=clad, media=[clad, med], site_medium=site)
    h = get_handle(tolerance="tight")
    (_,), (ia,) = compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms, eps_dfreq=de, eps_d2freq=d2e)], handle=h,
                                      want_fields=False, return_info=True, derivatives=("freq2",))
    (_,), (ib,) = compute_modes_batch([dict(section=sec, coords=coords, freq=F0, mode_spec=ms)], handle=h, want_fields=False,
                                      return_info=True, derivatives=("freq2",))
    # the section's tables are central differences of eps(f) (1e-4 and 1e-3 relative steps: ~1e-8 and ~1e-6 errors)
    assert np.abs(ia["d2n_dfreq2"] - ib["d2n_dfreq2"]).max() <= 1e-5 * np.abs(ia["d2n_dfreq2"]).max()


def test_dispersion_changes_nothing_else_and_does_not_depend_on_the_batch():
    wl = W.si_strip(64, 2, W.sweep_freqs(64))
    eps = np.ascontiguousarray(np.stack(wl.eps_cross))
    probs = [dict(eps_cross=eps, coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec) for f in wl.freqs]
    h = get_handle()
    plain = compute_modes_batch(probs, handle=h)
    first, i1 = compute_modes_batch(probs, handle=h, return_info=True, derivatives=("freq", "eps"))
    second, i2 = compute_modes_batch(probs, handle=h, return_info=True, derivatives=("freq", "eps", "freq2"))
    for a, b, c, x, y in zip(plain, first, second, i1, i2):
        assert np.array_equal(a[1], c[1]) and np.array_equal(a[0], c[0]) and np.array_equal(b[1], c[1])
        assert np.array_equal(x["dn_dfreq"], y["dn_dfreq"]) and np.array_equal(x["dn_deps"], y["dn_deps"])
        assert np.all(np.isfinite(y["d2n_dfreq2"]))
    (alone,), (ia,) = compute_modes_batch([probs[17]], handle=h, return_info=True, derivatives=("freq2",))
    # one problem alone may stop at a different iterate of the eigen-solve and of its correction solves (within the tolerances)
    assert np.abs(ia["d2n_dfreq2"] - i2[17]["d2n_dfreq2"]).max() <= 1e-5 * np.abs(ia["d2n_dfreq2"]).max()


def test_near_degenerate_pml_pair_returns():
    fac, _, _ = GOLDEN_CASES["pml_none_128"]
    wl = fac()
    h = get_handle()
    tol = TOLERANCES["reference"]["inner_tol"]
    (_,), (info,) = compute_modes_batch([dict(eps_cross=wl.eps_cross, coords=wl.coords, freq=wl.freqs[0], mode_spec=wl.mode_spec)], handle=h,
                                        want_fields=False, return_info=True, derivatives=("freq2",))
    res, d2 = info["d2n_residual"], info["d2n_dfreq2"]
    assert np.all(np.isfinite(res))
    for m in range(d2.size):
        if np.isfinite(d2[m]):
            assert res[m] <= 100 * tol, (m, res[m])
        else:
            assert res[m] > 100 * tol, (m, res[m])


def test_scope():
    eps, coords, ms = _strip(48)
    h = get_handle()
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=dataclasses.replace(ms, angle_theta=0.2))], handle=h,
                            derivatives=("freq2",))
    basis = np.zeros((6, 48, 48, 1, ms.num_modes), complex)
    basis[0, 20:28, 20:28] = 1.0
    basis[1, 20:28, 20:28, 0, 1] = 1.0
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms, solver_basis_fields=basis)], handle=h, derivatives=("freq2",))
    pec = eps.copy()
    for c in (0, 4, 8):
        pec[c][:4] = -1e8
    mu = [np.ones((48, 48), complex) if k in (0, 4, 8) else np.zeros((48, 48), complex) for k in range(9)]
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=pec, coords=coords, freq=F0, mode_spec=ms, mu_cross=mu)], handle=h, derivatives=("freq2",))
