"""GPU: d n / df, the group index and the nine-component d n / d eps of tensorial modes (angled planes, off-diagonal eps) from the
transposed Krylov-Schur pass and the tensorial derivative kernels (csrc/derivatives.cuh tensor_deriv_*), against the float64 model
oracle/tensor_derivatives.py (its own right and left eigenvectors), against device finite differences, for material dispersion,
for invariance of everything else, for diagonal problems under the flag, and for the scope rules that stay."""
import dataclasses

import numpy as np
import pytest

from oracle import restatement as R
from oracle import tensor_derivatives as T
from tests import mg_cases
from tests.golden import cases as G
from tidy3d_b200 import plugin
from tidy3d_b200 import workloads as W
from tidy3d_b200.sections import Medium, Section
from tidy3d_b200.solver import compute_modes_batch, get_handle

pytestmark = pytest.mark.gpu
CASES = ["angled_48_minus", "lossy_angled_40", "lossy_angled_40_minus", "angle_bend_44", "offdiag_48", "angled_nonuniform_pml"]
DERIV = ("freq", "eps")
OBSERVED = {}


def _angled_nonuniform_pml():
    """Angled strip on a graded grid with PML: reciprocity does not give the left eigenvector here."""
    wl = G._nonuniform(48)
    wl.mode_spec = W.ModeSpecLike(num_modes=3, angle_theta=0.25, angle_phi=0.4, num_pml=(6, 6), target_neff=2.2)
    return wl, {}


def _case(name):
    return _angled_nonuniform_pml() if name == "angled_nonuniform_pml" else mg_cases.case(name)


def _problem(wl, kw, **over):
    p = dict(eps_cross=np.ascontiguousarray(np.stack([np.asarray(c, complex) for c in wl.eps_cross])), coords=wl.coords,
             freq=float(wl.freqs[0]), mode_spec=wl.mode_spec, **kw)
    p.update(over)
    return p


def _solve(probs, **kw):
    return compute_modes_batch(probs, handle=get_handle(tolerance="tight"), return_info=True, **kw)


def _observe(key, err):
    OBSERVED[key] = max(OBSERVED.get(key, 0.0), err)
    return err


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if OBSERVED:
        print("\nlargest errors:", {k: f"{v:.2e}" for k, v in sorted(OBSERVED.items())})


@pytest.mark.parametrize("name", CASES)
def test_device_matches_model(name):
    wl, kw = _case(name)
    p = _problem(wl, kw)
    (res,), (info,) = _solve([p], want_fields=False, derivatives=DERIV, left_solve=True)
    k = wl.mode_spec.num_modes
    assert info["left_paired"] == k
    assert info["dn_deps"].shape == (9, p["eps_cross"].shape[1], p["eps_cross"].shape[2], k)
    st = R.setup(wl.eps_cross, wl.coords, p["freq"], wl.mode_spec, kw.get("symmetry", (0, 0)), kw.get("mu_cross"))
    msign = -1.0 if (kw.get("direction") == "-" and R._is_complex(st["eps"])) else 1.0
    vals, u, _, w = T.eigenpairs(st, k + 2, tol=1e-13, msign=msign)  # two more: the device's k nearest may differ at the edge
    for m in range(k):
        q = int(np.argmin(np.abs(vals * st["knorm"] - res[1][m])))
        out = T.derivatives(wl.eps_cross, wl.coords, p["freq"], wl.mode_spec, u[:, q], w[:, q], kw.get("symmetry", (0, 0)),
                            kw.get("mu_cross"), msign=msign)
        assert abs(out["n"] - res[1][m]) <= 1e-7 * abs(out["n"])
        e_f = _observe(f"dn_dfreq {name}", abs(info["dn_dfreq"][m] - out["dn_dfreq"]) / abs(out["dn_dfreq"]))
        e_g = _observe(f"dn_deps {name}", np.abs(info["dn_deps"][..., m] - out["dn_deps_tensor"]).max() / np.abs(out["dn_deps_tensor"]).max())
        # ten times the largest errors measured on an H100 (DESIGN.md §6)
        assert e_f <= 3e-6 and e_g <= 5e-8, (m, e_f, e_g)


@pytest.mark.parametrize("name", ["angled_nonuniform_pml", "offdiag_48"])
def test_group_index_matches_device_finite_differences(name):
    wl, kw = _case(name)
    p = _problem(wl, kw)
    step = 1e-3
    freqs = [p["freq"] * (1 - step), p["freq"], p["freq"] * (1 + step)]
    res, _ = _solve([dict(p, freq=f) for f in freqs], want_fields=False)
    _, _, ng_fd, _ = plugin.group_index(np.array([r[1] for r in res]), freqs, step)
    _, (info,) = _solve([p], want_fields=False, derivatives=("freq",), left_solve=True)
    bound = 10 * step**2 + 10 * 1e-9 / step
    assert _observe(f"n_group {name}", np.abs(info["n_group"] - ng_fd[0]).max()) <= bound, (info["n_group"], ng_fd[0])


@pytest.mark.parametrize("comp", [0, 1, 2, 8])
def test_region_gradient_matches_device_finite_difference(comp):
    wl, kw = _case("angled_nonuniform_pml")
    p = _problem(wl, kw)
    eps = p["eps_cross"]
    core = eps[0].real > 5
    _, (info,) = _solve([p], want_fields=False, derivatives=("eps",), left_solve=True)
    delta = 1e-3 * np.abs(eps[:, core]).max()
    ep, em = eps.copy(), eps.copy()
    ep[comp] = ep[comp] + delta * core
    em[comp] = em[comp] - delta * core
    (rp, rm), _ = _solve([dict(p, eps_cross=ep), dict(p, eps_cross=em)], want_fields=False)
    fd = (rp[1] - rm[1]) / 2
    pred = delta * info["dn_deps"][comp][core].sum(axis=0)
    err = _observe(f"gradient fd {comp}", np.abs(pred - fd).max() / (np.abs(fd).max() + 1e-300))
    assert np.abs(pred - fd).max() <= 1e-3 * np.abs(fd).max() + 1e-8, (comp, pred, fd, err)


def _rotated(e, a):
    """the diagonal tensor diag(e) rotated by a about z: off-diagonal xy / yx"""
    c, s = np.cos(a), np.sin(a)
    Rm = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    return Rm @ np.diag(e) @ Rm.T


def test_dispersive_anisotropic_section():
    wl = W.angled(48, num_modes=2)
    eps = np.ascontiguousarray(np.stack(wl.eps_cross))
    f0 = float(wl.freqs[0])
    core_eps = eps[0].real.max()
    base = np.array([core_eps, 0.9 * core_eps, 1.05 * core_eps])
    clad = Medium(complex(eps[0].real.min()))
    core = Medium(lambda f: _rotated(base * (1 + 0.05 * (f / f0 - 1)), 0.3))
    site = np.stack([np.isclose(eps[c].real, core_eps) for c in (0, 4, 8)]).astype(np.uint16)
    sec = Section(background=clad, media=[clad, core], site_medium=site)
    step = 1e-3
    freqs = [f0 * (1 - step), f0, f0 * (1 + step)]
    res, _ = _solve([dict(section=sec, coords=wl.coords, freq=f, mode_spec=wl.mode_spec) for f in freqs], want_fields=False)
    _, _, ng_fd, _ = plugin.group_index(np.array([r[1] for r in res]), freqs, step)
    sp = dict(section=sec, coords=wl.coords, freq=f0, mode_spec=wl.mode_spec)
    _, (info,) = _solve([sp], want_fields=False, derivatives=DERIV, left_solve=True)
    bound = 10 * step**2 + 10 * 1e-9 / step + 1e-7  # + the O(1e-8) central difference of the medium's eps(f)
    assert _observe("n_group dispersive", np.abs(info["n_group"] - ng_fd[0]).max()) <= bound, (info["n_group"], ng_fd[0])
    # the same medium as an array, with and without its d eps / df
    e_arr = np.zeros((9,) + eps.shape[1:], complex)
    d_arr = np.zeros_like(e_arr)
    t0, t1 = core.tensor(f0), core.dtensor_dfreq(f0)
    for kk, (r, c) in enumerate((r, c) for r in range(3) for c in range(3)):
        m = site[r].astype(bool)  # eps_r* is sampled at the E_r site
        e_arr[kk] = np.where(m, t0[r, c], clad.tensor(f0)[r, c])
        d_arr[kk] = np.where(m, t1[r, c], 0.0)
    ap = dict(eps_cross=e_arr, coords=wl.coords, freq=f0, mode_spec=wl.mode_spec)
    _, (ia,) = _solve([dict(ap, eps_dfreq=d_arr)], want_fields=False, derivatives=DERIV, left_solve=True)
    _, (ind,) = _solve([ap], want_fields=False, derivatives=DERIV, left_solve=True)
    assert np.abs(ia["n_group"] - info["n_group"]).max() <= 1e-9 * np.abs(info["n_group"]).max()
    assert np.abs(ind["n_group"] - info["n_group"]).min() > 100 * bound  # the material term matters here


def test_nothing_else_changes_and_batch_position():
    wl = W.angled(48, num_modes=2)
    eps = np.ascontiguousarray(np.stack(wl.eps_cross))
    ms = dataclasses.replace(wl.mode_spec, num_pml=(6, 6))
    probs = [dict(eps_cross=eps, coords=wl.coords, freq=float(f), mode_spec=ms) for f in W.sweep_freqs(16)]
    h = get_handle()
    plain, ip = compute_modes_batch(probs, handle=h, return_info=True)
    withd, iw = compute_modes_batch(probs, handle=h, return_info=True, derivatives=DERIV, left_solve=True)
    for a, b, x, y in zip(plain, withd, ip, iw):
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[0], b[0])
        for key in ("converged", "restarts", "op_applies", "inner_iters"):
            assert x[key] == y[key], key
        assert y["left_paired"] == 2 and x["left_paired"] == -1
    (_,), (ia,) = compute_modes_batch([probs[5]], handle=h, return_info=True, derivatives=DERIV, left_solve=True)
    assert np.abs(ia["dn_dfreq"] - iw[5]["dn_dfreq"]).max() <= 1e-5 * np.abs(ia["dn_dfreq"]).max()


def test_diagonal_problems_under_the_flag():
    wl = W.si_strip(64, 2)
    ms = dataclasses.replace(wl.mode_spec, num_pml=(8, 8))
    p = dict(eps_cross=np.ascontiguousarray(np.stack(wl.eps_cross)), coords=wl.coords, freq=float(wl.freqs[0]), mode_spec=ms)
    h = get_handle()
    (_,), (a,) = compute_modes_batch([p], handle=h, return_info=True, want_fields=False, derivatives=DERIV)
    (_,), (b,) = compute_modes_batch([p], handle=h, return_info=True, want_fields=False, derivatives=DERIV, left_solve=True)
    assert np.array_equal(a["dn_dfreq"], b["dn_dfreq"]) and np.array_equal(a["dn_deps"], b["dn_deps"])
    assert a["op_applies"] == b["op_applies"] and a["left_paired"] == b["left_paired"] == 2
    # the nine-row layout through the binding directly: off-diagonal rows zero, diagonal rows those of dn_deps
    from tidy3d_b200 import _cabi

    pk = _cabi.PackedProblem(p["eps_cross"], p["coords"], p["freq"], ms, left_solve=True)
    with h.lock:
        rc, _, _, res = h.solve_batch([pk], want_fields=False, want_dfreq=True, want_deps_tensor=True)
        full = h.last_dn_deps[0]
    assert rc == _cabi.OK and res[0].left_paired == 2
    assert np.array_equal(full[[0, 4, 8]], a["dn_deps"]) and not np.any(full[[1, 2, 3, 5, 6, 7]])


def test_scope_under_the_flag():
    wl = W.angled(48, num_modes=2)
    p = dict(eps_cross=np.ascontiguousarray(np.stack(wl.eps_cross)), coords=wl.coords, freq=float(wl.freqs[0]), mode_spec=wl.mode_spec)
    h = get_handle()
    for d in (("freq2",), ("group_eps",), ("freq3",)):
        with pytest.raises(NotImplementedError):
            compute_modes_batch([p], handle=h, derivatives=d, left_solve=True)
    with pytest.raises(NotImplementedError, match="left_solve=True"):
        compute_modes_batch([p], handle=h, derivatives=("freq",))
    basis = np.zeros((6, 48, 48, 1, 2), complex)
    basis[0, 20:28, 20:28] = 1.0
    basis[1, 20:28, 20:28, 0, 1] = 1.0
    ms0 = dataclasses.replace(wl.mode_spec, angle_theta=0.0)
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(p, mode_spec=ms0, solver_basis_fields=basis)], handle=h, derivatives=DERIV, left_solve=True)
    pec = p["eps_cross"].copy()
    for c in (0, 4, 8):
        pec[c][:4] = -1e8
    mu = [np.ones((48, 48), complex) if k in (0, 4, 8) else np.zeros((48, 48), complex) for k in range(9)]
    with pytest.raises(NotImplementedError):
        compute_modes_batch([dict(p, mode_spec=ms0, eps_cross=pec, mu_cross=mu)], handle=h, derivatives=("freq",), left_solve=True)
