"""GPU: the perturbation responses (derivatives "pert", "group_pert", "disp_pert"; deriv_pert_kernel, tensor_pert_kernel and the
PERT variants of group_grad_kernel / disp_grad_kernel in csrc/derivatives.cuh) against einsum over the maps the same call
delivers, against device finite differences of n_group and the dispersion, for a section's per-medium table against the same
scene as arrays, for batching and sharing, for bit-identical other outputs, for the NaN rule and for the rejected scope."""
import dataclasses

import numpy as np
import pytest

from tests.golden.cases import CASES as GOLDEN_CASES
from tests.test_gpu_mode_dispersion import CASES, F0, _problem, _strip
from tests.test_gpu_tensor_derivatives import _case as _tensor_case
from tests.test_gpu_tensor_derivatives import _problem as _tensor_problem
from tidy3d_b200 import plugin
from tidy3d_b200 import workloads as W
from tidy3d_b200.sections import Medium, Section
from tidy3d_b200.solver import TOLERANCES, compute_modes_batch, get_handle

pytestmark = pytest.mark.gpu
# |response - einsum(map, delta eps)| / einsum(|map|, |delta eps|): 10 x the largest value measured on an H100 (DESIGN.md §6)
EINSUM_RTOL = 3.5e-14
PAIRS = (("dn_dpert", "dn_deps"), ("d2n_dfreq_dpert", "d2n_dfreq_deps"), ("d2n_dfreq2_dpert", "d2n_dfreq2_deps"))


def _perts(eps, npml=0):
    """(3, 9, Nx, Ny): a real core-only change, a complex change that covers the PML cells, and a zz-only anisotropic one."""
    core = eps[0].real > 5
    nx, ny = core.shape
    edge = np.zeros_like(core)
    w = max(npml, 6)
    edge[:w], edge[-w:], edge[:, :w], edge[:, -w:] = True, True, True, True
    out = np.zeros((3, 9, nx, ny), complex)
    for c in (0, 4, 8):
        out[0, c] = core
        out[1, c] = (0.3 - 0.7j) * edge + 0.2j * core
    out[2, 8] = core
    return out


def _check_against_maps(info, pert, comps, kinds):
    err = 0.0
    for key, mkey in PAIRS[:kinds]:
        got, mp = info[key], info[mkey]
        want = np.einsum("axym,kaxy->km", mp, pert[:, comps])
        scale = np.einsum("axym,kaxy->km", np.abs(np.nan_to_num(mp)), np.abs(pert[:, comps]))
        nan = np.isnan(mp).any(axis=(0, 1, 2))
        assert np.array_equal(np.isnan(got), np.broadcast_to(nan, got.shape)), key
        ok = ~np.isnan(got)
        e = float(np.max(np.abs(got - want)[ok] / scale[ok])) if ok.any() else 0.0
        print(f"[pert] {key}: largest |response - einsum| / einsum(|map|, |delta eps|) = {e:.3e}")
        assert e <= EINSUM_RTOL, (key, e)
        err = max(err, e)
    return err


@pytest.mark.parametrize("name", sorted(CASES))
def test_responses_match_einsum_over_the_maps(name):
    p = _problem(name)
    npml = max(getattr(p["mode_spec"], "num_pml", (0, 0)))
    pert = _perts(p["eps_cross"], npml)
    p["eps_pert"] = pert
    (_,), (info,) = compute_modes_batch([p], handle=get_handle(tolerance="tight"), want_fields=False, return_info=True,
                                        derivatives=("disp_eps", "disp_pert"))
    assert info["dn_dpert"].shape == (3, p["mode_spec"].num_modes)
    _check_against_maps(info, pert, [0, 4, 8], 3)
    assert np.array_equal(info["dng_dpert"], info["dn_dpert"].real + F0 * info["d2n_dfreq_dpert"].real)
    assert np.array_equal(info["dispersion_dpert"], plugin.dispersion_gradient_of(F0, info["d2n_dfreq_dpert"], info["d2n_dfreq2_dpert"]))


@pytest.mark.parametrize("name", ["angled_nonuniform_pml", "offdiag_48"])
def test_tensorial_responses_match_einsum_over_the_nine_row_map(name):
    wl, kw = _tensor_case(name)
    p = _tensor_problem(wl, kw)
    rng = np.random.default_rng(7)
    pert = rng.standard_normal((2, 9) + p["eps_cross"].shape[1:]) + 1j * rng.standard_normal((2, 9) + p["eps_cross"].shape[1:])
    p["eps_pert"] = pert
    (_,), (info,) = compute_modes_batch([p], handle=get_handle(tolerance="tight"), want_fields=False, return_info=True,
                                        derivatives=("eps", "pert"), left_solve=True)
    _check_against_maps(info, pert, list(range(9)), 1)


def _fd(make, pert, deltas=(2e-2, 1e-2)):
    """dng_dpert and dispersion_dpert at delta 0 against central differences of the device's n_group and dispersion under
    eps + delta * pert (make(delta) -> problem), Richardson-bounded over the two steps."""
    h = get_handle(tolerance="tight")
    p0 = make(0.0)
    p0["eps_pert"] = pert
    (_,), (info,) = compute_modes_batch([p0], handle=h, want_fields=False, return_info=True, derivatives=("disp_pert",))
    for key, fkey in (("dng_dpert", "n_group"), ("dispersion_dpert", "dispersion")):
        got = info[key][0]
        fds = []
        for d in deltas:
            _, infos = compute_modes_batch([make(d), make(-d)], handle=h, want_fields=False, return_info=True, derivatives=("freq2",))
            fds.append((infos[0][fkey] - infos[1][fkey]) / (2 * d))
        noise = 1e-6 * np.abs(info[fkey]) if fkey == "dispersion" else 1e-9 * np.abs(info[fkey])
        bound = 2 * np.abs(fds[0] - fds[1]) + 2 * noise / deltas[1]
        print(f"[pert] {key}: analytic {got}, fd {fds[1]}, bound {bound}")
        assert np.all(np.abs(got - fds[1]) <= bound), (key, got, fds, bound)
        assert np.all(bound <= 0.05 * np.abs(got)), (key, got, bound)  # the check is not vacuous


def test_strip_responses_match_device_finite_differences():
    eps, coords, ms = _strip(64)
    core = eps[0].real > 5
    pert = np.zeros((1, 9) + core.shape, complex)
    for c in (0, 4, 8):
        pert[0, c] = core

    def make(d):
        return dict(eps_cross=eps + d * pert[0], coords=coords, freq=F0, mode_spec=ms)

    _fd(make, pert)


def test_curved_section_complex_response_matches_device_finite_differences():
    eps, coords, ms = _strip(64)
    core_eps = complex(eps[0].real.max())
    clad = Medium(complex(eps[0].real.min()))
    site = np.stack([np.isclose(eps[c].real, core_eps.real) for c in (0, 4, 8)]).astype(np.uint16)
    dz = 1 + 0.2j  # a complex change of the core medium, at fixed d eps / df and d^2 eps / df^2
    media = {}

    def make(d):
        core = Medium(lambda f: core_eps * (1 + 0.05 * (f / F0 - 1) + 0.2 * (f / F0 - 1) ** 2) + d * dz)
        media[d] = core
        return dict(section=Section(background=clad, media=[clad, core], site_medium=site), coords=coords, freq=F0, mode_spec=ms)

    h = get_handle(tolerance="tight")
    p0 = make(0.0)
    p0["eps_pert"] = [{media[0.0]: dz}]
    (_,), (info,) = compute_modes_batch([p0], handle=h, want_fields=False, return_info=True, derivatives=("disp_pert",))
    for key, fkey in (("dng_dpert", "n_group"), ("dispersion_dpert", "dispersion")):
        got, fds = info[key][0], []
        for d in (2e-2, 1e-2):
            _, infos = compute_modes_batch([make(d), make(-d)], handle=h, want_fields=False, return_info=True, derivatives=("freq2",))
            fds.append((infos[0][fkey] - infos[1][fkey]) / (2 * d))
        noise = 1e-6 * np.abs(info[fkey]) if fkey == "dispersion" else 1e-9 * np.abs(info[fkey])
        bound = 2 * np.abs(fds[0] - fds[1]) + 2 * noise / 1e-2
        print(f"[pert] curved section {key}: analytic {got}, fd {fds[1]}, bound {bound}")
        assert np.all(np.abs(got - fds[1]) <= bound), (key, got, fds, bound)
        assert np.all(bound <= 0.05 * np.abs(got)), (key, got, bound)


def test_section_table_matches_the_same_scene_as_arrays():
    eps, coords, ms = _strip(64)
    core_eps, clad_eps = complex(eps[0].real.max()), complex(eps[0].real.min())
    clad, core = Medium(clad_eps), Medium(core_eps)
    site = np.stack([np.isclose(eps[c].real, core_eps.real) for c in (0, 4, 8)]).astype(np.uint16)
    arr_eps = np.zeros_like(eps)  # the section's scene sampled as arrays
    pert = np.zeros((1, 9) + eps.shape[1:], complex)
    for a, c in enumerate((0, 4, 8)):
        arr_eps[c] = np.where(site[a] == 1, core_eps, clad_eps)
        pert[0, c] = site[a] == 1
    h = get_handle(tolerance="tight")
    sec = dict(section=Section(background=clad, media=[clad, core], site_medium=site), coords=coords, freq=F0, mode_spec=ms,
               eps_pert=[{core: 1.0}])
    arr = dict(eps_cross=arr_eps, coords=coords, freq=F0, mode_spec=ms, eps_pert=pert)
    _, (i_sec, i_arr) = compute_modes_batch([sec, arr], handle=h, want_fields=False, return_info=True, derivatives=("group_eps", "group_pert"))
    _check_against_maps(i_sec, pert, [0, 4, 8], 2)  # the rasterised table is the core mask
    for key in ("dn_dpert", "d2n_dfreq_dpert"):  # the same coefficient fields: the same bits
        assert np.array_equal(i_sec[key], i_arr[key]), (key, np.abs(i_sec[key] - i_arr[key]).max())


def test_batching_sharing_and_batch_position():
    wl = W.si_strip(64, 2, W.sweep_freqs(64))
    eps = np.ascontiguousarray(np.stack(wl.eps_cross))
    core = eps[0].real > 5
    rng = np.random.default_rng(3)
    p5 = np.zeros((5, 9) + core.shape, complex)
    for c in (0, 4, 8):
        p5[:, c] = rng.standard_normal((5,) + core.shape) * core + 0.1j * rng.standard_normal((5,) + core.shape)
    h = get_handle()
    kinds = ("disp_pert",)

    def probs(ep, copies=False):
        return [dict(eps_cross=eps, coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec, eps_pert=ep.copy() if copies else ep) for f in wl.freqs]

    _, shared = compute_modes_batch(probs(p5), handle=h, want_fields=False, return_info=True, derivatives=kinds)
    _, copied = compute_modes_batch(probs(p5, copies=True), handle=h, want_fields=False, return_info=True, derivatives=kinds)
    keys = ("dn_dpert", "d2n_dfreq_dpert", "d2n_dfreq2_dpert")
    for a, b in zip(shared, copied):
        for key in keys:
            assert np.array_equal(a[key], b[key], equal_nan=True), key
    for k in (0, 3):
        _, one = compute_modes_batch(probs(np.ascontiguousarray(p5[k : k + 1])), handle=h, want_fields=False, return_info=True, derivatives=kinds)
        for a, b in zip(shared, one):
            for key in keys:
                assert np.array_equal(a[key][k], b[key][0], equal_nan=True), (k, key)
    pa = probs(p5)[17]
    (_,), (alone,) = compute_modes_batch([pa], handle=h, want_fields=False, return_info=True, derivatives=kinds)
    # one problem alone may stop at a different iterate of the eigen-solve and of its correction solves (within the tolerances)
    for key in keys:
        err = np.abs(alone[key] - shared[17][key]).max() / np.abs(alone[key]).max()
        print(f"[pert] alone against batch position 17, {key}: {err:.3e}")
        assert err <= 1e-3, (key, err)


def test_many_perturbations_in_launch_chunks_and_device_groups():
    """K = 17: the first-order scans take the perturbations in three launches of kPertGroup = 6, and the device holds
    kPertHeld = 16 at once, so the last one is gathered in a second device group (per mode slot in the dispersion pass).
    Every response is the bits of the same perturbation asked for alone."""
    wl = W.si_strip(64, 2, W.sweep_freqs(8))
    eps = np.ascontiguousarray(np.stack(wl.eps_cross))
    core = eps[0].real > 5
    rng = np.random.default_rng(11)
    p17 = np.zeros((17, 9) + core.shape, complex)
    for c in (0, 4, 8):
        p17[:, c] = rng.standard_normal((17,) + core.shape) * core + 0.1j * rng.standard_normal((17,) + core.shape)
    h = get_handle()

    def run(ep):
        probs = [dict(eps_cross=eps, coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec, eps_pert=ep) for f in wl.freqs]
        return compute_modes_batch(probs, handle=h, want_fields=False, return_info=True, derivatives=("disp_pert",))[1]

    many = run(p17)
    for k in (0, 5, 6, 12, 15, 16):
        one = run(np.ascontiguousarray(p17[k : k + 1]))
        for a, b in zip(many, one):
            for key in ("dn_dpert", "d2n_dfreq_dpert", "d2n_dfreq2_dpert"):
                assert np.array_equal(a[key][k], b[key][0], equal_nan=True), (k, key)


def test_pert_kinds_change_nothing_else():
    wl = W.si_strip(64, 2, W.sweep_freqs(64))
    eps = np.ascontiguousarray(np.stack(wl.eps_cross))
    pert = _perts(eps)
    probs = [dict(eps_cross=eps, coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec) for f in wl.freqs]
    h = get_handle()
    base, i1 = compute_modes_batch(probs, handle=h, return_info=True, derivatives=("disp_eps",))
    for p in probs:
        p["eps_pert"] = pert
    full, i2 = compute_modes_batch(probs, handle=h, return_info=True, derivatives=("disp_eps", "disp_pert"))
    keys = ("dn_dfreq", "n_group", "dn_deps", "d2n_dfreq2", "d2n_residual", "dispersion", "d2n_dfreq_deps", "dng_deps", "d3n_dfreq3",
            "dispersion_slope", "beta3", "d4n_dfreq4", "d4n_residual", "beta4", "d2n_dfreq2_deps", "dispersion_deps")
    for a, b, x, y in zip(base, full, i1, i2):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        for k in keys:
            assert np.array_equal(x[k], y[k], equal_nan=True), k
        assert np.all(np.isfinite(y["d2n_dfreq2_dpert"]))


def test_nan_where_the_maps_are():
    fac, _, _ = GOLDEN_CASES["pml_none_128"]
    wl = fac()
    eps = np.ascontiguousarray(np.stack([np.asarray(c, complex) for c in wl.eps_cross]))
    p = dict(eps_cross=eps, coords=wl.coords, freq=wl.freqs[0], mode_spec=wl.mode_spec, eps_pert=_perts(eps))
    (_,), (info,) = compute_modes_batch([p], handle=get_handle(), want_fields=False, return_info=True, derivatives=("disp_eps", "disp_pert"))
    tol = TOLERANCES["reference"]["inner_tol"]
    print(f"[pert] pml_none_128: d2n NaN {np.isnan(info['d2n_dfreq2']).tolist()}, d4n NaN {np.isnan(info['d4n_dfreq4']).tolist()}")
    for key, mkey in PAIRS:
        nan = np.isnan(info[mkey]).all(axis=(0, 1, 2))
        assert np.array_equal(np.isnan(info[key]).all(axis=0), nan) and np.array_equal(np.isnan(info[key]).any(axis=0), nan), key
    assert np.array_equal(np.isnan(info["d2n_dfreq_dpert"][0]), info["d2n_residual"] > 100 * tol)


def test_scope():
    eps, coords, ms = _strip(48)
    pert = _perts(eps)
    h = get_handle()
    angled = dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=dataclasses.replace(ms, angle_theta=0.2), eps_pert=pert)
    with pytest.raises(NotImplementedError, match="left_solve=True"):
        compute_modes_batch([angled], handle=h, derivatives=("pert",))
    for kind in ("group_pert", "disp_pert"):
        for left in (False, True):
            with pytest.raises(NotImplementedError):
                compute_modes_batch([angled], handle=h, derivatives=(kind,), left_solve=left)
    basis = np.zeros((6, 48, 48, 1, ms.num_modes), complex)
    basis[0, 20:28, 20:28] = 1.0
    basis[1, 20:28, 20:28, 0, 1] = 1.0
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=eps, coords=coords, freq=F0, mode_spec=ms, solver_basis_fields=basis, eps_pert=pert)], handle=h,
                            derivatives=("pert",))
    pec = eps.copy()
    for c in (0, 4, 8):
        pec[c][:4] = -1e8
    mu = [np.ones((48, 48), complex) if k in (0, 4, 8) else np.zeros((48, 48), complex) for k in range(9)]
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(eps_cross=pec, coords=coords, freq=F0, mode_spec=ms, mu_cross=mu, eps_pert=pert)], handle=h,
                            derivatives=("pert",))
