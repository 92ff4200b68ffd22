"""CPU: the perturbation responses.  The float64 model (oracle/mode_perturbation.py: the oracle's gradient maps contracted
against delta eps_k) against central differences of the dense eigenpair's n under eps +- h delta eps on the group-gradient case
set, for a real core-only, a complex PML-covering and a zz-only perturbation, and on the tensorial adjoint cases for nine-component
ones; plugin.dispersion_gradient_of on (K, M) responses; the b200ms_pert binding and the argument errors, without a device."""
import dataclasses
import re

import numpy as np
import pytest

from oracle import mode_derivatives as D
from oracle import mode_dispersion as MD
from oracle import mode_dispersion_gradient as DG
from oracle import mode_perturbation as MP
from oracle import restatement as R
from oracle import tensor_derivatives as T
from tests import mg_cases
from tests.test_mode_derivatives_cpu import F0, _operator, _track
from tests.test_mode_dispersion_cpu import CASES2, _inputs, _setup
from tidy3d_b200 import _cabi, plugin
from tidy3d_b200 import workloads as W
from tidy3d_b200.sections import Medium, Section
from tidy3d_b200.solver import compute_modes_batch


def _perts(c):
    """A real core-only change, a complex change of the core and of a band of cells next to the PML, and a zz-only one (cells
    inside the PML are covered by the device test against the delivered maps)."""
    core = np.asarray(c["core"], bool)
    px, py = (getattr(c["ms"], "num_pml", None) or (0, 0))
    band = np.zeros_like(core)
    band[px : px + 2, py:-py or None] = True
    band[-px - 2 : (-px or None), py:-py or None] = True
    band[px:-px or None, py : py + 2] = True
    band[px:-px or None, -py - 2 : (-py or None)] = True
    out = np.zeros((3, 9) + core.shape, complex)
    for a in (0, 4, 8):
        out[0, a] = core
        out[1, a] = (0.3 - 0.7j) * (band & ~core) + 0.2j * core
    out[2, 8] = core
    return out


def _fundamental(c):
    lam, V = np.linalg.eig(_operator(c, F0))
    m = int(np.argmin(lam.real))
    return lam[m], V[:, m]


@pytest.mark.parametrize("name", sorted(CASES2))
def test_first_order_response_matches_dense_central_difference(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    eps0 = c["eps_at"](F0)
    out = D.derivatives(eps0, (c["x"], c["y"]), F0, c["ms"], v, lam, c["sym"], c["mu"])
    got = MP.contract(out["dn_deps"], _perts(c))
    knorm = R.setup(eps0, (c["x"], c["y"]), F0, c["ms"], c["sym"], c["mu"])["knorm"]

    def n_at(pert, h):
        eps = [np.asarray(e, complex) + h * pert[i] for i, e in enumerate(eps0)]
        lh = _track(_operator(c, F0, eps), lam)
        return np.sqrt(-lh + 0j) * knorm * np.sign(np.sqrt(-lh + 0j).real)

    for k, pert in enumerate(_perts(c)):
        def cd(h):
            return (n_at(pert, h) - n_at(pert, -h)) / (2 * h)

        h = 1e-3
        a, b = cd(h), cd(h / 2)
        bound = 2 * abs(a - b) + 1e-8 * abs(got[k])  # + the dense eigenvalue's roundoff over the step
        print(f"[pert cpu] {name} pert {k}: model {got[k]:.6e}, fd {b:.6e}, bound {bound:.1e}")
        assert abs(got[k] - b) <= bound, (k, got[k], b, bound)


@pytest.mark.parametrize("name", sorted(CASES2))
def test_second_order_responses_match_dense_central_differences(name):
    """The group and dispersion maps of the model contracted against delta eps_k against central differences, under
    eps +- h delta eps at fixed d eps / df and d^2 eps / df^2, of the exact n' and n'' of the dense eigenpair."""
    c = _setup(name)
    lam, v = _fundamental(c)
    de, d2e = _inputs(c)
    eps0 = c["eps_at"](F0)
    coords = (c["x"], c["y"])
    out = DG.dispersion_gradient(eps0, coords, F0, c["ms"], v, lam, c["sym"], c["mu"], eps_dfreq=de, eps_d2freq=d2e)
    perts = _perts(c)
    got = {"dn_dfreq": MP.contract(out["d2n_dfreq_deps"], perts), "d2n_dfreq2": MP.contract(out["d2n_dfreq2_deps"], perts)}

    def derivs(pert, h):
        eps = [np.asarray(e, complex) + h * pert[i] for i, e in enumerate(eps0)]
        lh, V = np.linalg.eig(_operator(c, F0, eps))
        m = int(np.argmin(np.abs(lh - lam)))
        o = MD.second_derivatives(eps, coords, F0, c["ms"], V[:, m], lh[m], c["sym"], c["mu"], eps_dfreq=de, eps_d2freq=d2e)
        return o["dn_dfreq"], o["d2n_dfreq2"]

    for k, pert in enumerate(perts):
        d = {}
        for h in (1e-3, 5e-4):
            p, q = derivs(pert, h), derivs(pert, -h)
            d[h] = [(p[j] - q[j]) / (2 * h) for j in range(2)]
        for j, key in enumerate(("dn_dfreq", "d2n_dfreq2")):
            a, b, g = d[1e-3][j], d[5e-4][j], got[key][k]
            bound = 2 * abs(a - b) + 1e-7 * abs(g)  # + the dense model's roundoff over the step
            print(f"[pert cpu] {name} pert {k} d({key}): model {g:.6e}, fd {b:.6e}, bound {bound:.1e}")
            assert abs(g - b) <= bound, (k, key, g, b, bound)


@pytest.mark.parametrize("name", ["angled_48_minus", "offdiag_48"])
def test_tensorial_response_matches_dense_central_difference(name):
    wl, kw = mg_cases.case(name)
    st = R.setup(wl.eps_cross, wl.coords, float(wl.freqs[0]), wl.mode_spec, kw.get("symmetry", (0, 0)), kw.get("mu_cross"))
    msign = -1.0 if (kw.get("direction") == "-" and R._is_complex(st["eps"])) else 1.0
    vals, u, _, w = T.eigenpairs(st, 1, tol=1e-13, msign=msign)
    out = T.derivatives(wl.eps_cross, wl.coords, float(wl.freqs[0]), wl.mode_spec, u[:, 0], w[:, 0], kw.get("symmetry", (0, 0)),
                        kw.get("mu_cross"), msign=msign)
    rng = np.random.default_rng(5)
    shape = np.asarray(wl.eps_cross[0]).shape
    pert = (rng.standard_normal((2, 9) + shape) + 1j * rng.standard_normal((2, 9) + shape)) * 0.1
    got = MP.contract(out["dn_deps_tensor"], pert, comps=range(9))

    def n_at(p, h):
        eps = [np.asarray(e, complex) + h * p[i] for i, e in enumerate(wl.eps_cross)]
        s = R.setup(eps, wl.coords, float(wl.freqs[0]), wl.mode_spec, kw.get("symmetry", (0, 0)), kw.get("mu_cross"))
        v2, _, _, _ = T.eigenpairs(s, 3, tol=1e-13, msign=msign)
        return v2[np.argmin(np.abs(v2 - vals[0]))] * s["knorm"]

    for k in range(2):
        def cd(h):
            return (n_at(pert[k], h) - n_at(pert[k], -h)) / (2 * h)

        a, b = cd(1e-3), cd(5e-4)
        bound = 2 * abs(a - b) + 1e-8 * abs(got[k])  # + the dense eigenvalue's roundoff over the step
        print(f"[pert cpu] {name} pert {k}: model {got[k]:.6e}, fd {b:.6e}, bound {bound:.1e}")
        assert abs(got[k] - b) <= bound, (k, got[k], b, bound)


def test_dispersion_gradient_of_takes_k_by_m_responses():
    rng = np.random.default_rng(1)
    f = W.C_0 / 1.55
    a = rng.standard_normal((4, 3)) + 1j * rng.standard_normal((4, 3))
    b = (rng.standard_normal((4, 3)) + 1j * rng.standard_normal((4, 3))) * 1e-15
    want = np.array([[plugin.dispersion_gradient_of(f, a[k, m], b[k, m]) for m in range(3)] for k in range(4)])
    assert np.array_equal(plugin.dispersion_gradient_of(f, a, b), want)
    assert np.array_equal(MP.dispersion_response(f, a, b), want)


def test_pert_struct_mirrors_the_header():
    src = open(_cabi.os.path.join(_cabi._HERE, "..", "include", "b200ms.h")).read()
    body = src[: src.index("} b200ms_pert;")].rsplit("typedef struct {", 1)[1]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = re.findall(r"(\w+);", body)
    assert names == [n for n, _ in _cabi.Pert._fields_]
    assert "b200ms_solve_batch_ext3" in _cabi.EXPORTS and "int b200ms_solve_batch_ext3(" in src


def _strip_problem(**over):
    wl = W.si_strip(24, 2)
    p = dict(eps_cross=np.ascontiguousarray(np.stack(wl.eps_cross)), coords=wl.coords, freq=float(wl.freqs[0]), mode_spec=wl.mode_spec)
    p.update(over)
    return p


def test_argument_errors_need_no_device():
    p = _strip_problem()
    pert = np.zeros((2, 9, 24, 24), complex)
    with pytest.raises(ValueError, match="no problem gives it"):
        compute_modes_batch([p], derivatives=("group_pert",))
    with pytest.raises(ValueError, match="ask for one of them"):
        compute_modes_batch([dict(p, eps_pert=pert)], derivatives=("eps",))
    with pytest.raises(ValueError, match="eps_pert must have shape"):
        compute_modes_batch([dict(p, eps_pert=pert[:, :, :23])], derivatives=("pert",))
    with pytest.raises(ValueError, match="need a 'section'"):
        compute_modes_batch([dict(p, eps_pert=[{Medium(2.0): 1.0}])], derivatives=("pert",))
    clad, core = Medium(2.1), Medium(12.0)
    sec = Section(background=clad, media=[clad, core], site_medium=np.zeros((3, 24, 24), np.uint16))
    sp = dict(section=sec, coords=p["coords"], freq=p["freq"], mode_spec=p["mode_spec"])
    with pytest.raises(ValueError, match="not part of the section"):
        compute_modes_batch([dict(sp, eps_pert=[{Medium(3.0): 1.0}])], derivatives=("pert",))
    with pytest.raises(ValueError, match="sequence of dicts"):
        compute_modes_batch([dict(sp, eps_pert=pert)], derivatives=("pert",))
    with pytest.raises(ValueError, match="sequence of dicts"):
        compute_modes_batch([dict(sp, eps_pert=[])], derivatives=("pert",))


def test_one_eps_pert_object_on_two_grids_is_checked_per_problem():
    small = _strip_problem()
    wl = W.si_strip(32, 2)
    big = dict(eps_cross=np.ascontiguousarray(np.stack(wl.eps_cross)), coords=wl.coords, freq=float(wl.freqs[0]), mode_spec=wl.mode_spec)
    x = np.zeros((2, 9, 24, 24), complex)
    with pytest.raises(ValueError, match="eps_pert must have shape"):  # shared with a 24x24 problem first, then a 32x32 one
        compute_modes_batch([dict(small, eps_pert=x), dict(big, eps_pert=x)], derivatives=("pert",))


def test_section_table_follows_the_medium_order():
    clad, core = Medium(2.1), Medium(12.0)
    sec = Section(background=clad, media=[clad, core])
    t = sec.pert_table([{core: 1.0}, {clad: (1, 2, 3), core: np.eye(3) * 0.5j}])
    assert t.shape == (2, 2, 9)
    assert np.array_equal(t[0, 1], np.eye(3).ravel()) and not t[0, 0].any()
    assert np.array_equal(t[1, 0], np.diag([1, 2, 3]).ravel().astype(complex)) and np.array_equal(t[1, 1], 0.5j * np.eye(3).ravel())
