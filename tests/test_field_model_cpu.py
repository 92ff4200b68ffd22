"""CPU: the field-recovery model oracle/field_model.py against the restatement, so that the GPU tests of the device epilogue
(test_gpu_field_epilogue.py) compare it with a pinned model.

a. On the golden cases the restatement's own modes (tol 1e-12) go in: the model reproduces all six components the restatement
   delivers, whose fields the goldens pin to the reference.
b. On O(1) random vectors, which weigh the boundary, wall and PML rows that guided modes leave near zero, the model matches the
   restatement's expressions written with its assembled sparse difference matrices (Q v, Dxf / Dyf, the q-form Ez, J^T).
c. The permutation, the direction signs and the conjugate flip on hand-made inputs.

Errors are scaled by the model's sum of absolute values of each entry's terms."""
import numpy as np
import pytest

from oracle import field_model as FM
from oracle import mg_model as M
from oracle import restatement as R
from tests.golden import cases as G

CASES = ["c1_64", "c1_64_minus", "c1_64_sym_pmc_pec", "nonuniform_56", "lossy_48", "c4_96", "c4_96_axis0", "mu_cross_40", "slab1d_x1",
         "slab1d_y1", "angled_48_minus", "offdiag_48", "lossy_angled_40", "lossy_angled_40_minus"]  # fmt: skip
PEC_CASES = ["pec_block_40", "pec_split_40"]
# Largest scaled errors: 6.5e-14 (Ez of c4_96_axis0, where the restatement's q-form difference iez (Dxb Hy - Dyb Hx) cancels),
# 8e-16 elsewhere.  Next to a PEC-model eps of 1 + 1e8 i the q-form cancels terms of size 1e8 |v|, but the u-form's own term
# sum holds the same 1e8 |v| (|exx| |v1|), so the PEC cases stay within the one bound (7.9e-15 measured).
TOL = 1e-12


def _case(name):
    fac, kw, _ = G.CASES[name]
    wl = fac()
    kw = G.resolve_kwargs(wl, kw)
    return wl, kw


def _problem(wl, kw):
    eps = wl.eps_cross
    split = kw.get("split_curl_scaling")
    if split is not None:  # compute_modes divides eps by the scaling first (solver.py:122-124)
        eps = [np.array(e, complex) for e in eps]
        for comp, idx in enumerate((0, 4, 8)):
            out = ~np.isclose(split[comp], 0)
            eps[idx][out] /= np.asarray(split[comp])[out]
    st = R.setup(eps, wl.coords, wl.freqs[0], wl.mode_spec, kw.get("symmetry", (0, 0)), kw.get("mu_cross"))
    incidence = kw.get("mu_cross") is not None or split is not None
    return M.Problem(st, incidence=incidence, num_modes=wl.mode_spec.num_modes)


def _err(F, ref, S):
    S = np.asarray(S)
    floor = 1e-300 + 1e-30 * S.reshape(2, 3, -1).max(axis=2)[:, :, None, None, None]
    return float((np.abs(np.asarray(F) - ref) / (S + floor)).max())


_SOLVED = {}


def _solved(name):
    if name not in _SOLVED:
        wl, kw = _case(name)
        f, n, spec = R.compute_modes(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, tol=1e-12, **kw)
        _SOLVED[name] = (wl, kw, f[:, :, :, :, 0, :], n, spec)
    return _SOLVED[name]


@pytest.mark.parametrize("name", CASES + PEC_CASES)
def test_model_reproduces_the_restatement_modes(name):
    wl, kw, f, n, spec = _solved(name)
    prob = _problem(wl, kw)
    direction = kw.get("direction", "+")
    assert prob.tensorial == spec.startswith("tensorial")
    v = FM.vectors(prob, f, direction)
    F, S = FM.fields(prob, v, n / prob.st["knorm"], direction=direction)
    split = kw.get("split_curl_scaling")
    if split is not None:  # solver.py:904-919 (identity where the scaling is 1)
        sc = np.asarray(split)
        F[0] = F[0] / np.where(np.isclose(sc, 0), 1.0, sc)[..., None] * (~np.isclose(sc, 0))[..., None]
    e = _err(F, f, S)
    assert e <= TOL, (name, e)


def _reference_fields(prob, v, n, direction):
    """The restatement's expressions (compute_modes) with its assembled matrices, on any vectors."""
    st, N = prob.st, prob.nx * prob.ny
    dxf, dxb, dyf, dyb = R.d_matrices(st)
    e, m = st["eps"], st["mu"]
    v = np.asarray(v, complex).T
    hs = -1j / R.ETA_0
    if not prob.tensorial:
        if prob.masked:  # the incidence formulation: 1 / eps_zz zeroed on PEC cells, eps_xx / eps_yy unknowns removed
            iez = prob.fields[2].ravel()
        else:
            iez = 1 / e[2, 2]
        _, qmat, _ = R.assemble_diagonal(st)
        inv = 1 / (1j * np.asarray(n))
        hq = (qmat @ v) * inv
        hx, hy = hq[:N], hq[N:]
        hz = (dxf @ v[N:] - dyf @ v[:N]) / m[2, 2][:, None]
        ez = (dxb @ hy - dyb @ hx) * iez[:, None]
        E = np.stack((v[:N], v[N:], ez))
        H = np.stack((hx, hy, hz)) * hs
        if direction == "-":
            H[0] *= -1
            H[1] *= -1
            E[2] *= -1
    else:
        ex, ey, hx, hy = v[:N], v[N : 2 * N], v[2 * N : 3 * N], v[3 * N :]
        hz = (dxf @ ey - dyf @ ex - m[2, 0][:, None] * hx - m[2, 1][:, None] * hy) / m[2, 2][:, None]
        ez = (dxb @ hy - dyb @ hx - e[2, 0][:, None] * ex - e[2, 1][:, None] * ey) / e[2, 2][:, None]
        E, H = np.stack((ex, ey, ez)), np.stack((hx, hy, hz)) * hs
        if FM.conj_flip(prob, direction):
            E, H = np.conj(E), -np.conj(H)
    E = np.einsum("ijn,inm->jnm", st["jac_e"], E)
    H = np.einsum("ijn,inm->jnm", st["jac_h"], H)
    return np.stack((E, H)).reshape(2, 3, prob.nx, prob.ny, -1)


def _random_vectors(prob, k, rng):
    shape = (k, (4 if prob.tensorial else 2) * prob.nx * prob.ny)
    v = rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
    if prob.masked:  # removed PEC unknowns are zero (BatchSolver::mask_E)
        v = v * np.concatenate((~prob.pec[0].ravel(), ~prob.pec[1].ravel()))[None, :]
    return v


@pytest.mark.parametrize("name", CASES + PEC_CASES + ["pec_block_40_mu"])
def test_model_matches_the_assembled_expressions_on_random_vectors(name):
    if name == "pec_block_40_mu":
        from tests import mg_cases

        wl, kw = mg_cases.case(name)
    else:
        wl, kw = _case(name)
    prob = _problem(wl, kw)
    assert prob.masked == (name in ("pec_split_40", "pec_block_40_mu"))
    rng = np.random.default_rng(5)
    k = 3
    v = _random_vectors(prob, k, rng)
    n = rng.uniform(1.2, 3.0, k) + 1j * rng.uniform(-0.1, 0.1, k)
    for direction in ("+", "-"):
        F, S = FM.fields(prob, v, n, direction=direction)
        ref = _reference_fields(prob, v, n, direction)
        e = _err(F, ref, S)
        assert e <= TOL, (name, direction, e)
        # random vectors carry weight on the first and last rows and columns: none of them is zero there
        for c in range(3):
            for edge in (F[0, c, 0], F[0, c, -1], F[1, c, :, 0], F[1, c, :, -1]):
                if c < 2 or (prob.nx > 1 and prob.ny > 1):
                    assert np.abs(edge).max() > 0


def test_permutation_picks_the_slot_of_each_output_mode():
    wl, kw = _case("lossy_48")
    prob = _problem(wl, kw)
    rng = np.random.default_rng(1)
    v = _random_vectors(prob, 3, rng)
    n = np.array([2.1 + 0.01j, 1.9 - 0.02j, 1.5 + 0.0j])
    perm = [2, 0, 1]
    F, S = FM.fields(prob, v, n, perm=perm)
    for q, s in enumerate(perm):
        Fq, Sq = FM.fields(prob, v[s : s + 1], n[q : q + 1])
        assert np.array_equal(F[..., q], Fq[..., 0]) and np.array_equal(S[..., q], Sq[..., 0])
    # n belongs to the output mode, not to the slot: Ez and the in-plane H scale with 1 / n
    G, _ = FM.fields(prob, v, n[[1, 2, 0]], perm=perm)
    assert np.allclose(G[0, 2] * n[[1, 2, 0]], F[0, 2] * n, rtol=1e-14, atol=0)
    assert np.array_equal(G[1, 2], F[1, 2]) and np.array_equal(G[0, :2], F[0, :2])
    for p in ([0, 1, 2], perm):
        assert np.array_equal(FM.vectors(prob, FM.fields(prob, v, n, perm=p)[0]), v[p])


@pytest.mark.parametrize("name, flip", [("angled_48_minus", True), ("lossy_angled_40_minus", False), ("c1_64_minus", False)])
def test_direction_signs_and_the_conjugate_flip(name, flip):
    wl, kw = _case(name)
    prob = _problem(wl, kw)
    assert FM.conj_flip(prob, "-") == flip and not FM.conj_flip(prob, "+")
    rng = np.random.default_rng(2)
    v = _random_vectors(prob, 2, rng)
    n = np.array([1.8 + 0.01j, 1.6 + 0.0j])
    Fp, _ = FM.fields(prob, v, n, direction="+")
    Fm, _ = FM.fields(prob, v, n, direction="-")
    if not prob.tensorial:  # Hx, Hy and Ez change sign (before the bend scale, which is linear)
        sign = np.array([[1, 1, -1], [-1, -1, 1]])[:, :, None, None, None]
        assert np.array_equal(Fm, sign * Fp)
    elif flip:  # tensorial_real: E = conj(E), H = -conj(H), then J^T (real)
        assert np.allclose(Fm[0], np.conj(Fp[0]), rtol=1e-15, atol=0) and np.allclose(Fm[1], -np.conj(Fp[1]), rtol=1e-15, atol=0)
        assert np.array_equal(Fm[:, :2], np.stack((np.conj(Fp[0, :2]), -np.conj(Fp[1, :2]))))
    else:  # tensorial_complex: the sign lives in the operator (its eigenvalue), not in the recovery
        assert np.array_equal(Fm, Fp)
    assert np.allclose(FM.vectors(prob, Fm, "-"), v, rtol=1e-15, atol=0)
