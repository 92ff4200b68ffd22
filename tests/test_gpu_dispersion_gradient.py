"""GPU: the dispersion gradient of the fourth-order pass (disp_grad_kernel, csrc/derivatives.cuh) against the float64 model
(oracle/mode_dispersion_gradient.py) on the device's own eigenvectors, against device finite differences of the dispersion (also
for a section with curved eps(f)), for bit-identical other outputs and batch invariance, for the NaN rule of the two correction
solves, and for the rejected scope."""
import dataclasses

import numpy as np
import pytest

from oracle import mode_dispersion_gradient as DG
from tests.golden.cases import CASES as GOLDEN_CASES
from tests.test_gpu_mode_dispersion import CASES, F0, _problem, _strip
from tidy3d_b200 import plugin
from tidy3d_b200 import workloads as W
from tidy3d_b200.sections import Medium, Section
from tidy3d_b200.solver import TOLERANCES, compute_modes_batch, get_handle

pytestmark = pytest.mark.gpu
# device against the model on the device's own eigenvectors (tight preset), max |map - model| / max |model| per mode
# 10 x the largest error measured on an H100 80GB HBM3 (700 W limit): 1.42e-8 on plain_64 (pml_96 and minus_96: 4.5e-10)
MODEL_RTOL = 1.5e-7


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_matches_model_on_its_own_eigenvectors(name):
    p = _problem(name)
    h = get_handle(tolerance="tight")
    (res,), (info,) = compute_modes_batch([p], handle=h, return_info=True, derivatives=("disp_eps",))
    fields, n = res[0], res[1]
    errs = []
    for m in range(p["mode_spec"].num_modes):
        v = np.r_[fields[0, 0, :, :, 0, m].ravel(), fields[0, 1, :, :, 0, m].ravel()]
        out = DG.dispersion_gradient(list(p["eps_cross"]), p["coords"], p["freq"], p["mode_spec"], v, -(n[m] ** 2), p["symmetry"])
        got = info["d2n_dfreq2_deps"][..., m]
        errs.append(np.abs(got - out["d2n_dfreq2_deps"]).max() / np.abs(out["d2n_dfreq2_deps"]).max())
        want = plugin.dispersion_gradient_of(p["freq"], info["d2n_dfreq_deps"][..., m], got)
        assert np.array_equal(info["dispersion_deps"][..., m], want)
    print(f"[disp_eps] {name}: max relative |d2n_dfreq2_deps - model| = {max(errs):.3e}")
    assert max(errs) <= MODEL_RTOL, errs


def _fd_region(make, region, deltas=(2e-2, 1e-2)):
    """sum over `region` (3, Nx, Ny) of the device's dispersion_deps at delta 0 against the central difference of the device's
    dispersion under eps +- delta on that region (make(delta) -> problem), Richardson-bounded over the two steps."""
    h = get_handle(tolerance="tight")
    (_,), (info,) = compute_modes_batch([make(0.0)], handle=h, want_fields=False, return_info=True, derivatives=("disp_eps",))
    got = np.array([np.sum(info["dispersion_deps"][a][region[a]], axis=0) for a in range(3)]).sum(axis=0)
    fds = []
    for d in deltas:
        _, infos = compute_modes_batch([make(d), make(-d)], handle=h, want_fields=False, return_info=True, derivatives=("freq2",))
        fds.append((infos[0]["dispersion"] - infos[1]["dispersion"]) / (2 * d))
    noise = 1e-6 * np.abs(info["dispersion"])  # the dispersion of the tight preset to about 1e-7 relative
    bound = 2 * np.abs(fds[0] - fds[1]) + 2 * noise / deltas[1]
    print(f"[disp_eps] region: analytic {got}, fd {fds[1]}, bound {bound}")
    assert np.all(np.abs(got - fds[1]) <= bound), (got, fds, bound)
    assert np.all(bound <= 0.05 * np.abs(got)), (got, bound)  # the check is not vacuous
    return got, bound


def test_region_gradient_matches_device_finite_difference():
    eps, coords, ms = _strip(64)
    core = eps[0].real > 5
    region = np.stack([core, np.zeros_like(core), np.zeros_like(core)])

    def make(d):
        e = eps.copy()
        e[0] = e[0] + d * core
        return dict(eps_cross=e, coords=coords, freq=F0, mode_spec=ms)

    _fd_region(make, region)


def test_curved_dispersive_section_region_gradient():
    eps, coords, ms = _strip(64)
    core_eps = complex(eps[0].real.max())
    clad = Medium(complex(eps[0].real.min()))
    site = np.stack([np.isclose(eps[c].real, core_eps.real) for c in (0, 4, 8)]).astype(np.uint16)

    def make(d):  # a constant shift of the core medium keeps d eps / df and d^2 eps / df^2
        core = Medium(lambda f: core_eps * (1 + 0.05 * (f / F0 - 1) + 0.2 * (f / F0 - 1) ** 2) + d)
        return dict(section=Section(background=clad, media=[clad, core], site_medium=site), coords=coords, freq=F0, mode_spec=ms)

    got, bound = _fd_region(make, site == 1)
    # the material terms matter here: the same core without dispersion gives another gradient
    h = get_handle(tolerance="tight")
    (_,), (nd,) = compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms)], handle=h, want_fields=False,
                                      return_info=True, derivatives=("disp_eps",))
    plain = np.array([np.sum(nd["dispersion_deps"][a][site[a] == 1], axis=0) for a in range(3)]).sum(axis=0)
    print(f"[disp_eps] curved section: {got}, nondispersive {plain}, bound {bound}")
    assert np.all(np.abs(plain - got) > bound), (plain, got, bound)


def test_disp_eps_changes_nothing_else_and_does_not_depend_on_the_batch():
    wl = W.si_strip(64, 2, W.sweep_freqs(64))
    eps = np.ascontiguousarray(np.stack(wl.eps_cross))
    probs = [dict(eps_cross=eps, coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec) for f in wl.freqs]
    h = get_handle()
    base, i1 = compute_modes_batch(probs, handle=h, return_info=True, derivatives=("group_eps", "freq4"))
    full, i2 = compute_modes_batch(probs, handle=h, return_info=True, derivatives=("disp_eps",))
    keys = ("dn_dfreq", "dn_deps", "d2n_dfreq2", "d2n_residual", "dispersion", "d2n_dfreq_deps", "dng_deps", "d3n_dfreq3",
            "dispersion_slope", "beta3", "d4n_dfreq4", "d4n_residual", "beta4")
    for a, b, x, y in zip(base, full, i1, i2):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        for k in keys:
            assert np.array_equal(x[k], y[k], equal_nan=True), k
        assert np.all(np.isfinite(y["d2n_dfreq2_deps"])) and np.abs(y["d2n_dfreq2_deps"]).max() > 0
    (alone,), (ia,) = compute_modes_batch([probs[17]], handle=h, return_info=True, derivatives=("disp_eps",))
    # one problem alone may stop at a different iterate of the eigen-solve and of its correction solves (within the tolerances)
    err = np.abs(ia["d2n_dfreq2_deps"] - i2[17]["d2n_dfreq2_deps"]).max() / np.abs(ia["d2n_dfreq2_deps"]).max()
    print(f"[disp_eps] alone against batch position 17: {err:.3e}")
    assert err <= 1e-3


def test_maps_are_nan_where_d4n_is():
    fac, _, _ = GOLDEN_CASES["pml_none_128"]
    wl = fac()
    h = get_handle()
    (_,), (info,) = compute_modes_batch([dict(eps_cross=wl.eps_cross, coords=wl.coords, freq=wl.freqs[0], mode_spec=wl.mode_spec)], handle=h,
                                        want_fields=False, return_info=True, derivatives=("disp_eps",))
    tol = TOLERANCES["reference"]["inner_tol"]
    stopped = (info["d2n_residual"] > 100 * tol) | (info["d4n_residual"] > 100 * tol)
    print(f"[disp_eps] pml_none_128: d4n NaN {np.isnan(info['d4n_dfreq4']).tolist()}")
    assert np.array_equal(np.isnan(info["d4n_dfreq4"]), stopped)
    for m in range(stopped.size):
        for k in ("d2n_dfreq2_deps", "dispersion_deps"):
            mp = info[k][..., m]
            assert np.all(np.isnan(mp)) if stopped[m] else np.all(np.isfinite(mp)), (k, m)


def test_scope():
    eps, coords, ms = _strip(48)
    h = get_handle()
    angled = dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=dataclasses.replace(ms, angle_theta=0.2))
    for left in (False, True):
        with pytest.raises(NotImplementedError):
            compute_modes_batch([angled], handle=h, derivatives=("disp_eps",), left_solve=left)
    basis = np.zeros((6, 48, 48, 1, ms.num_modes), complex)
    basis[0, 20:28, 20:28] = 1.0
    basis[1, 20:28, 20:28, 0, 1] = 1.0
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms, solver_basis_fields=basis)], handle=h,
                            derivatives=("disp_eps",))
    pec = eps.copy()
    for c in (0, 4, 8):
        pec[c][:4] = -1e8
    mu = [np.ones((48, 48), complex) if k in (0, 4, 8) else np.zeros((48, 48), complex) for k in range(9)]
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=pec, coords=coords, freq=F0, mode_spec=ms, mu_cross=mu)], handle=h, derivatives=("disp_eps",))
