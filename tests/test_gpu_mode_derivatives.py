"""GPU: d n / df, the group index and d n / d eps of the derivative pass (csrc/derivatives.cuh) against the float64 model
(oracle/mode_derivatives.py) on the device's own eigenvectors, against device finite differences, and for batch invariance."""
import dataclasses

import numpy as np
import pytest

from oracle import mode_derivatives as D
from tidy3d_b200 import plugin
from tidy3d_b200 import workloads as W
from tidy3d_b200.sections import Medium, Section
from tidy3d_b200.solver import compute_modes_batch, get_handle

pytestmark = pytest.mark.gpu
F0 = W.C_0 / 1.55


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
    "minus_single_128": dict(n=128, direction="-", spec=dict(num_pml=(10, 10), precision="single")),
}


def _problem(name):
    c = CASES[name]
    eps, coords, ms = _strip(c["n"], **c.get("spec", {}))
    if c.get("lossy"):
        eps = _lossy(eps)
    return dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms, symmetry=c.get("sym", (0, 0)), direction=c.get("direction", "+"))


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_matches_model_on_its_own_eigenvectors(name):
    p = _problem(name)
    if p["mode_spec"].precision == "single":  # the model needs the fp64 vectors: take them from a double-precision twin
        p_model = dict(p, mode_spec=dataclasses.replace(p["mode_spec"], precision="double"))
    else:
        p_model = p
    h = get_handle(tolerance="tight")
    (res,), (info,) = compute_modes_batch([p], handle=h, return_info=True, derivatives=("freq", "eps"))
    (res_d,), (info_d,) = compute_modes_batch([p_model], handle=h, return_info=True, derivatives=("freq", "eps"))
    fields, n = res_d[0], res_d[1]
    nx, ny = p["eps_cross"].shape[1:]
    for m in range(p["mode_spec"].num_modes):
        v = np.r_[fields[0, 0, :, :, 0, m].ravel(), fields[0, 1, :, :, 0, m].ravel()]
        out = D.derivatives(list(p["eps_cross"]), p["coords"], p["freq"], p["mode_spec"], v, -(n[m] ** 2), p["symmetry"])
        for inf in (info, info_d):
            assert abs(inf["dn_dfreq"][m] - out["dn_dfreq"]) <= 1e-9 * abs(out["dn_dfreq"]), (m, inf["dn_dfreq"][m], out["dn_dfreq"])
            err = np.abs(inf["dn_deps"][..., m] - out["dn_deps"]).max()
            assert err <= 1e-9 * np.abs(out["dn_deps"]).max(), (m, err)
        assert info["dn_deps"].shape == (3, nx, ny, 2)


@pytest.mark.parametrize("name", ["pml_96", "bend_lossy_64"])
def test_group_index_matches_device_finite_differences(name):
    p = _problem(name)
    h = get_handle(tolerance="tight")
    step = 1e-3
    freqs = [F0 * (1 - step), F0, F0 * (1 + step)]
    res = compute_modes_batch([dict(p, freq=f) for f in freqs], handle=h, want_fields=False)
    _, _, ng_fd, _ = plugin.group_index(np.array([r[1] for r in res]), freqs, step)
    (_,), (info,) = compute_modes_batch([p], handle=h, want_fields=False, return_info=True, derivatives=("freq",))
    # truncation of the central difference ~ n f^2 step^2 |n'''| (order 1e-6 here) plus the eigenvalue tolerance over the step
    bound = 10 * step**2 + 10 * 1e-9 / step
    assert np.abs(info["n_group"] - ng_fd[0]).max() <= bound, (info["n_group"], ng_fd[0])


def test_region_gradient_matches_device_finite_difference():
    p = _problem("pml_96")
    h = get_handle(tolerance="tight")
    eps = p["eps_cross"]
    core = eps[0].real > 5
    (_,), (info,) = compute_modes_batch([p], handle=h, want_fields=False, return_info=True, derivatives=("eps",))
    delta = 1e-3 * eps[0][core].real.max()
    ep, em = eps.copy(), eps.copy()
    for c in (0, 4, 8):
        ep[c] = ep[c] + delta * core
        em[c] = em[c] - delta * core
    (rp, rm) = compute_modes_batch([dict(p, eps_cross=ep), dict(p, eps_cross=em)], handle=h, want_fields=False)
    fd = (rp[1] - rm[1]) / 2
    pred = delta * info["dn_deps"][:, core, :].sum(axis=(0, 1))
    # second-order truncation ~ delta^2 |n''| plus the eigenvalue tolerance
    assert np.abs(pred - fd).max() <= 1e-3 * np.abs(fd).max() + 1e-8, (pred, fd)


def test_dispersive_section_group_index():
    eps, coords, ms = _strip(64)
    core_eps = complex(eps[0].real.max())
    clad = Medium(complex(eps[0].real.min()))
    core = Medium(lambda f: core_eps * (1 + 0.05 * (f / F0 - 1)))
    site = np.stack([np.isclose(eps[c].real, core_eps.real) for c in (0, 4, 8)]).astype(np.uint16)
    sec = Section(background=clad, media=[clad, core], site_medium=site)
    h = get_handle(tolerance="tight")
    step = 1e-3
    freqs = [F0 * (1 - step), F0, F0 * (1 + step)]
    res = compute_modes_batch([dict(section=sec, coords=coords, freq=f, mode_spec=ms) for f in freqs], handle=h, want_fields=False)
    _, _, ng_fd, _ = plugin.group_index(np.array([r[1] for r in res]), freqs, step)
    (_,), (info,) = compute_modes_batch([dict(section=sec, coords=coords, freq=F0, mode_spec=ms)], handle=h, want_fields=False,
                                        return_info=True, derivatives=("freq",))
    (_,), (info_nd,) = compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms)], handle=h, want_fields=False,
                                           return_info=True, derivatives=("freq",))
    bound = 10 * step**2 + 10 * 1e-9 / step + 1e-7  # + the O(1e-8) central difference of the medium's eps(f)
    assert np.abs(info["n_group"] - ng_fd[0]).max() <= bound, (info["n_group"], ng_fd[0])
    assert np.abs(info["n_group"] - info_nd["n_group"]).min() > 100 * bound  # the material term matters here


def test_derivatives_change_nothing_else_and_do_not_depend_on_the_batch():
    wl = W.si_strip(64, 2, W.sweep_freqs(64))
    eps = np.ascontiguousarray(np.stack(wl.eps_cross))
    probs = [dict(eps_cross=eps, coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec) for f in wl.freqs]
    h = get_handle()
    plain = compute_modes_batch(probs, handle=h)
    withd, infos = compute_modes_batch(probs, handle=h, return_info=True, derivatives=("freq", "eps"))
    for a, b in zip(plain, withd):
        assert np.array_equal(a[1], b[1])
        assert np.array_equal(a[0], b[0])
    (alone,), (ia,) = compute_modes_batch([probs[17]], handle=h, return_info=True, derivatives=("freq", "eps"))
    # the eigen-solve of one problem alone may stop at a different iterate than inside the batch (within eig_tol); the
    # derivatives follow the eigenpair, not the batch
    assert np.abs(ia["dn_dfreq"] - infos[17]["dn_dfreq"]).max() <= 1e-5 * np.abs(ia["dn_dfreq"]).max()
    if np.array_equal(alone[1], withd[17][1]):
        assert np.abs(ia["dn_dfreq"] - infos[17]["dn_dfreq"]).max() <= 1e-12 * np.abs(ia["dn_dfreq"]).max()


def test_scope():
    eps, coords, ms = _strip(48)
    h = get_handle()
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=dataclasses.replace(ms, angle_theta=0.2))], handle=h,
                            derivatives=("freq",))
    basis = np.zeros((6, 48, 48, 1, ms.num_modes), complex)
    basis[0, 20:28, 20:28] = 1.0
    basis[1, 20:28, 20:28, 0, 1] = 1.0
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms, solver_basis_fields=basis)], handle=h, derivatives=("eps",))
    pec = eps.copy()
    for c in (0, 4, 8):
        pec[c][:4] = -1e8
    mu = [np.ones((48, 48), complex) if k in (0, 4, 8) else np.zeros((48, 48), complex) for k in range(9)]
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=pec, coords=coords, freq=F0, mode_spec=ms, mu_cross=mu)], handle=h, derivatives=("freq",))
    with pytest.raises(ValueError):
        compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms)], handle=h, derivatives=("dispersion",))
    (res,), (info,) = compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms)], handle=h, want_fields=False,
                                          return_info=True, derivatives=("freq", "eps"))
    assert res[0] is None and np.all(np.isfinite(info["dn_dfreq"])) and np.abs(info["dn_deps"]).max() > 0
