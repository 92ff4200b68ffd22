"""GPU: the group-index gradient of the dispersion pass (group_grad_kernel, csrc/derivatives.cuh) against the float64 model
(oracle/mode_group_gradient.py) on the device's own eigenvectors, against device finite differences of n_group (also for a
dispersive section), for bit-identical other outputs, for the NaN rule of the correction solve, and for the rejected scope."""
import dataclasses

import numpy as np
import pytest

from oracle import mode_group_gradient as MG
from tests.golden.cases import CASES as GOLDEN_CASES
from tests.test_gpu_mode_dispersion import CASES, F0, _problem, _strip
from tidy3d_b200 import workloads as W
from tidy3d_b200.sections import Medium, Section
from tidy3d_b200.solver import TOLERANCES, compute_modes_batch, get_handle

pytestmark = pytest.mark.gpu
# device against the model on the device's own eigenvectors (tight preset), max |map - model| / max |model| per mode:
# 10 x the largest error measured on an H100 80GB HBM3 (700 W limit): 2.6e-8 on plain_64 (pml_96 and minus_96: 6.4e-10)
MODEL_RTOL = 2.6e-7


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_matches_model_on_its_own_eigenvectors(name):
    p = _problem(name)
    h = get_handle(tolerance="tight")
    (res,), (info,) = compute_modes_batch([p], handle=h, return_info=True, derivatives=("group_eps",))
    fields, n = res[0], res[1]
    errs = []
    for m in range(p["mode_spec"].num_modes):
        v = np.r_[fields[0, 0, :, :, 0, m].ravel(), fields[0, 1, :, :, 0, m].ravel()]
        out = MG.group_gradient(list(p["eps_cross"]), p["coords"], p["freq"], p["mode_spec"], v, -(n[m] ** 2), p["symmetry"])
        got = info["d2n_dfreq_deps"][..., m]
        errs.append(np.abs(got - out["d2n_dfreq_deps"]).max() / np.abs(out["d2n_dfreq_deps"]).max())
        assert np.array_equal(info["dng_deps"][..., m], info["dn_deps"][..., m].real + p["freq"] * got.real)
    print(f"[group_eps] {name}: max relative |d2n_dfreq_deps - model| = {max(errs):.3e}")
    assert max(errs) <= MODEL_RTOL, errs


def _fd_region(make, region, deltas=(2e-2, 1e-2)):
    """sum over `region` (3, Nx, Ny) of the device's dng_deps at delta 0 against the central difference of the device's
    n_group under eps +- delta on that region (make(delta) -> problem), Richardson-bounded over the two steps."""
    h = get_handle(tolerance="tight")
    (_,), (info,) = compute_modes_batch([make(0.0)], handle=h, want_fields=False, return_info=True, derivatives=("group_eps",))
    got = np.array([np.sum(info["dng_deps"][a][region[a]], axis=0) for a in range(3)]).sum(axis=0)
    fds = []
    for d in deltas:
        _, infos = compute_modes_batch([make(d), make(-d)], handle=h, want_fields=False, return_info=True, derivatives=("freq",))
        fds.append((infos[0]["n_group"] - infos[1]["n_group"]) / (2 * d))
    eig = 4e-9  # n_group of the tight preset to a few 1e-9
    bound = 2 * np.abs(fds[0] - fds[1]) + 2 * eig / deltas[1]
    print(f"[group_eps] region: analytic {got}, fd {fds[1]}, bound {bound}")
    assert np.all(np.abs(got - fds[1]) <= bound), (got, fds, bound)
    assert np.all(bound <= 0.05 * np.abs(got)), (got, bound)  # the check is not vacuous
    return got


def test_region_gradient_matches_device_finite_difference():
    eps, coords, ms = _strip(64)
    core = eps[0].real > 5
    region = np.stack([core, np.zeros_like(core), np.zeros_like(core)])

    def make(d):
        e = eps.copy()
        e[0] = e[0] + d * core
        return dict(eps_cross=e, coords=coords, freq=F0, mode_spec=ms)

    _fd_region(make, region)


def test_dispersive_section_region_gradient():
    eps, coords, ms = _strip(64)
    core_eps = complex(eps[0].real.max())
    clad = Medium(complex(eps[0].real.min()))
    site = np.stack([np.isclose(eps[c].real, core_eps.real) for c in (0, 4, 8)]).astype(np.uint16)

    def make(d):  # a constant shift of the core medium keeps d eps / df
        core = Medium(lambda f: core_eps * (1 + 0.05 * (f / F0 - 1) + 0.2 * (f / F0 - 1) ** 2) + d)
        return dict(section=Section(background=clad, media=[clad, core], site_medium=site), coords=coords, freq=F0, mode_spec=ms)

    got = _fd_region(make, site == 1)
    # the material term matters here: the same core without dispersion gives another gradient
    h = get_handle(tolerance="tight")
    (_,), (nd,) = compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms)], handle=h, want_fields=False,
                                      return_info=True, derivatives=("group_eps",))
    plain = np.array([np.sum(nd["dng_deps"][a][site[a] == 1], axis=0) for a in range(3)]).sum(axis=0)
    assert np.all(np.abs(plain - got) > 1e-3 * np.abs(got)), (plain, got)


def test_group_eps_changes_nothing_else():
    wl = W.si_strip(64, 2, W.sweep_freqs(64))
    eps = np.ascontiguousarray(np.stack(wl.eps_cross))
    probs = [dict(eps_cross=eps, coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec) for f in wl.freqs]
    h = get_handle()
    first, i1 = compute_modes_batch(probs, handle=h, return_info=True, derivatives=("freq", "eps", "freq2"))
    second, i2 = compute_modes_batch(probs, handle=h, return_info=True, derivatives=("group_eps",))
    for a, b, x, y in zip(first, second, i1, i2):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        for k in ("dn_dfreq", "dn_deps", "d2n_dfreq2", "d2n_residual"):
            assert np.array_equal(x[k], y[k]), k
        assert np.all(np.isfinite(y["d2n_dfreq_deps"])) and np.abs(y["d2n_dfreq_deps"]).max() > 0


def test_maps_are_nan_where_the_correction_solve_stopped():
    fac, _, _ = GOLDEN_CASES["pml_none_128"]
    wl = fac()
    h = get_handle()
    (_,), (info,) = compute_modes_batch([dict(eps_cross=wl.eps_cross, coords=wl.coords, freq=wl.freqs[0], mode_spec=wl.mode_spec)], handle=h,
                                        want_fields=False, return_info=True, derivatives=("group_eps",))
    tol = TOLERANCES["reference"]["inner_tol"]
    for m in range(info["d2n_dfreq2"].size):
        ok = info["d2n_residual"][m] <= 100 * tol
        assert np.isfinite(info["d2n_dfreq2"][m]) == ok
        assert (np.all(np.isfinite(info["d2n_dfreq_deps"][..., m])) if ok else np.all(np.isnan(info["d2n_dfreq_deps"][..., m])))


def test_scope():
    eps, coords, ms = _strip(48)
    h = get_handle()
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=dataclasses.replace(ms, angle_theta=0.2))], handle=h,
                            derivatives=("group_eps",))
    basis = np.zeros((6, 48, 48, 1, ms.num_modes), complex)
    basis[0, 20:28, 20:28] = 1.0
    basis[1, 20:28, 20:28, 0, 1] = 1.0
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms, solver_basis_fields=basis)], handle=h,
                            derivatives=("group_eps",))
    pec = eps.copy()
    for c in (0, 4, 8):
        pec[c][:4] = -1e8
    mu = [np.ones((48, 48), complex) if k in (0, 4, 8) else np.zeros((48, 48), complex) for k in range(9)]
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=pec, coords=coords, freq=F0, mode_spec=ms, mu_cross=mu)], handle=h, derivatives=("group_eps",))
