"""GPU: the field recovery (the epilogue) against the float64 model oracle/field_model.py, and the delivered modes against the
assembled operator.

Guided modes vanish at the domain edges, in the PML and at the walls, and the golden checks are overlaps and norms: a wrong
first or last row, a sign, a mode matched to the wrong n or slot would pass them.  So:

a. b200ms_debug_fields writes O(1) random vectors into the Ritz slots and runs the solver's own epilogue (per-problem
   permutation, DiagSite / TensorCell recovery, direction sign, conjugate flip, angled and bend back-transforms, complex128 or
   complex64 store).  Every batch position is compared with the model, and with the one-problem hook.
b. For solved goldens, the delivered fields are eigenvectors of the assembled float64 operator with the delivered n: the
   residual matches the device's max_residual, the model reproduces the six components from (Ex, Ey), n is sorted.
c. Delivery across device windows (max_batch 4, 11 distinct problems): every problem's fields pass b; pageable host arrays and
   torch device buffers receive the same bits; the post-processed fields are the raw ones times one scalar per mode, and the
   first problem of a window overlaps the last one of the previous window as the delivered fields say.

Errors are scaled by the model's sum of the absolute values of each entry's terms."""
import dataclasses

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import field_model as FM
from oracle import postprocess as OP
from oracle import restatement as R
from tests import mg_cases
from tidy3d_b200 import _cabi, compute_modes_batch
from tidy3d_b200 import workloads as W
from tidy3d_b200.solver import TOLERANCES

pytestmark = pytest.mark.gpu

CASES = ["c1_64", "c1_64_minus", "c1_64_sym_pmc_pec", "nonuniform_56", "lossy_48", "c4_96", "c4_96_axis0", "mu_cross_40",
         "pec_block_40_mu", "slab1d_x1", "slab1d_y1", "strip_75x131", "angled_48_minus", "offdiag_48", "lossy_angled_40",
         "lossy_angled_40_minus"]  # fmt: skip
GOLDEN = [c for c in CASES if c not in ("pec_block_40_mu", "strip_75x131")]
# About ten times the largest errors measured on an H100 80GB HBM3 at 700 W (OBSERVED is printed at the end): 1.1e-15 scaled
# (diagonal recovery in fp64; tensorial 3.4e-16, delivered modes 8.9e-16; complex64 outputs 7e-17 beyond their own rounding),
# and 0.36 for the residual agreement.
FP64_TOL = 1e-14
F32_ULP = 2.0**-23  # complex64 rounding of the stored value: half an ulp of each part, |.| <= 2^-24 sqrt(2) |F|
RES_TOL = 4.0  # |device - host residual| in units of eps_64 times the residual's rounding scale (see _residuals)
OBSERVED = {}


def _observe(key, err):
    OBSERVED[key] = max(OBSERVED.get(key, 0.0), err)
    return err


@pytest.fixture(scope="module")
def handle(built_lib):
    h = _cabi.Handle()
    yield h
    h.close()
    if OBSERVED:
        print("\nlargest scaled errors:", {k: f"{v:.2e}" for k, v in sorted(OBSERVED.items())})


def _workload(name, precision="double", num_modes=None):
    wl, kw = mg_cases.case(name)
    ms = dict(precision=precision)
    if num_modes is not None:
        ms["num_modes"] = num_modes
    wl.mode_spec = dataclasses.replace(wl.mode_spec, **ms)
    return wl, kw


def debug_fields(h, pks, vecs, n, perm):
    """b200ms_debug_fields: vecs (k, nb, len), n (nb, k) in solver units, perm (nb, k) -> (nb, 2, 3, nx, ny, k)."""
    p = pks[0].struct
    nb, k = len(pks), p.num_modes
    probs = (_cabi.Problem * nb)(*[pk.struct for pk in pks])
    out = np.empty((nb, 2, 3, p.nx, p.ny, k), np.complex64 if p.precision == 1 else complex)
    v = np.ascontiguousarray(vecs, complex)
    nn = np.ascontiguousarray(n, complex)
    pm = np.ascontiguousarray(perm, np.int32)
    rc = _cabi.lib().b200ms_debug_fields(h._h, nb, probs, _cabi._ptr(v.view(float)), _cabi._ptr(nn.view(float)),
                                         pm.ctypes.data_as(_cabi._ip), out.ctypes.data)
    assert rc == 0, (rc, h.last_error())
    return out


def _scaled(out, F, S, single):
    """max |out - F| / S, with the complex64 rounding of F allowed for single-precision output."""
    S = np.asarray(S)
    assert np.isfinite(out).all()
    if single:
        ref = F.astype(np.complex64).astype(complex)
        d = np.maximum(np.abs(out.astype(complex) - ref) - F32_ULP * np.abs(F), 0.0)
    else:
        d = np.abs(out - F)
    return float((d / (S + 1e-300)).max())


def check_batch(h, name, precision, nb, rng, num_modes=None):
    wl, kw = _workload(name, precision, num_modes)
    direction = kw.get("direction", "+")
    eps = np.ascontiguousarray(np.stack([np.asarray(e, complex) for e in wl.eps_cross]))
    freqs = [wl.freqs[0]] if nb == 1 else W.C_0 / np.linspace(1.5, 1.6, nb)  # a sweep sharing one medium
    pks = [mg_cases.packed(_cabi, wl, kw, freq=f, eps=eps) for f in freqs]
    probs = [mg_cases.model_problem(wl, kw, freq=f) for f in freqs]
    real = mg_cases.is_real(wl, kw)
    k = wl.mode_spec.num_modes
    L = (4 if probs[0].tensorial else 2) * probs[0].nx * probs[0].ny
    vecs = rng.standard_normal((k, nb, L)) + (0 if real else 1j * rng.standard_normal((k, nb, L)))
    n = rng.uniform(1.2, 3.0, (nb, k)) + 1j * rng.uniform(-0.1, 0.1, (nb, k))
    perm = np.array([rng.permutation(k) for _ in range(nb)])
    for b in range(nb):  # never the identity, and not the same at neighbouring positions
        while k > 1 and ((perm[b] == np.arange(k)).all() or (b and (perm[b] == perm[b - 1]).all() and k > 2)):
            perm[b] = rng.permutation(k)
    out = debug_fields(h, pks, vecs, n, perm)
    single = precision == "single"
    key = f"{'tensorial' if probs[0].tensorial else 'diagonal'} {precision}"
    for b in range(nb):
        F, S = FM.fields(probs[b], vecs[:, b], n[b], perm[b], direction)
        e = _observe(key, _scaled(out[b], F, S, single))
        assert e <= FP64_TOL, (name, precision, nb, b, e)
    for q in sorted({0, 1, nb - 1} & set(range(nb))):
        if nb > 1:  # the recovery is per cell: the same bits whatever the batch
            one = debug_fields(h, [pks[q]], vecs[:, q : q + 1], n[q : q + 1], perm[q : q + 1])
            assert np.array_equal(one[0], out[q]), (name, nb, q)
    return out


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("precision", ["double", "single"])
@pytest.mark.parametrize("nb", [1, 3])
def test_epilogue_matches_the_model(handle, name, precision, nb):
    check_batch(handle, name, precision, nb, np.random.default_rng(7 + nb))


@pytest.mark.parametrize("name", ["c1_64", "c4_96", "lossy_angled_40_minus"])
def test_epilogue_batch_of_64(handle, name):
    check_batch(handle, name, "double", 64, np.random.default_rng(64))


def test_epilogue_40_modes(handle):
    """Grid z = B M = 120 blocks, one per (problem, mode)."""
    check_batch(handle, "lossy_48", "double", 3, np.random.default_rng(40), num_modes=40)


def test_epilogue_rejects_a_non_permutation(handle):
    wl, kw = _workload("c1_64")
    pk = mg_cases.packed(_cabi, wl, kw)
    k, L = wl.mode_spec.num_modes, 2 * 64 * 64
    p = pk.struct
    probs = (_cabi.Problem * 1)(p)
    v = np.zeros((k, 1, L), complex)
    n = np.ones((1, k), complex)
    out = np.empty((2, 3, 64, 64, k), complex)
    pm = np.zeros((1, k), np.int32)
    rc = _cabi.lib().b200ms_debug_fields(handle._h, 1, probs, _cabi._ptr(v.view(float)), _cabi._ptr(n.view(float)),
                                         pm.ctypes.data_as(_cabi._ip), out.ctypes.data)
    assert rc == _cabi.ERR_ARG and "permutation" in handle.last_error()


# ---- b. delivered modes against the assembled operator ---------------------------------------------------------------------
def _operator(prob, direction):
    """The float64 operator whose eigenpairs the solver delivers, and its eigenvalue as a function of n (solver units)."""
    st = prob.st
    if not prob.tensorial:
        return R.assemble_diagonal(st)[2], lambda n: -(n**2)
    A = R.assemble_tensorial(st) * (-1j)
    if direction == "-" and FM.eps_complex(prob):  # solver.py:669-670
        A = A * -1
    return A.tocsr(), lambda n: n


def _residuals(prob, direction, v, n):
    """||A v - lambda v|| / (|lambda| ||v||) per mode, and the rounding scale of that ratio (|A| |v| + |lambda| |v|)."""
    A, lam_of = _operator(prob, direction)
    lam = lam_of(n)
    V = v.T
    r = A @ V - lam[None, :] * V
    absA = sp.csr_matrix((np.abs(A.data), A.indices, A.indptr), shape=A.shape)
    den = np.abs(lam) * np.linalg.norm(V, axis=0)
    scale = np.linalg.norm(absA @ np.abs(V) + np.abs(lam)[None, :] * np.abs(V), axis=0) / den
    return np.linalg.norm(r, axis=0) / den, scale


def check_delivered(prob, direction, f, n_complex, max_residual, key):
    f = np.asarray(f)[:, :, :, :, 0, :]
    k = f.shape[-1]
    assert (np.diff(n_complex.real) <= 0).all(), n_complex  # sorted by descending Re n
    n = n_complex / prob.st["knorm"]
    v = FM.vectors(prob, f, direction)
    F, S = FM.fields(prob, v, n, None, direction)
    e = _observe(f"delivered {key}", _scaled(f, F, S, f.dtype == np.complex64))
    assert e <= FP64_TOL, (key, e)
    if f.dtype == np.complex64:
        return  # the fields are rounded to complex64: their residual is that rounding, not the solve's
    res, scale = _residuals(prob, direction, v, n)
    assert res.shape == (k,)
    d = abs(res.max() - max_residual) / (np.finfo(float).eps * scale.max())
    _observe(f"residual / rounding {key}", d)
    assert d <= RES_TOL, (key, res.max(), max_residual, scale.max())


@pytest.fixture(scope="module")
def tight(built_lib):
    h = _cabi.Handle(**TOLERANCES["tight"])
    yield h
    h.close()


@pytest.mark.parametrize("name", GOLDEN)
def test_delivered_modes_are_eigenpairs_of_the_assembled_operator(tight, name):
    wl, kw = mg_cases.case(name)
    direction = kw.get("direction", "+")
    prob = mg_cases.model_problem(wl, kw)
    p = dict(eps_cross=wl.eps_cross, coords=wl.coords, freq=wl.freqs[0], mode_spec=wl.mode_spec, symmetry=kw.get("symmetry", (0, 0)),
             direction=direction, mu_cross=kw.get("mu_cross"))
    out, info = compute_modes_batch([p], handle=tight, return_info=True)
    f, n, _ = out[0]
    check_delivered(prob, direction, f, n, info[0]["max_residual"], name)


# ---- c. delivery across windows ----------------------------------------------------------------------------------------------
NPROB, MAX_BATCH = 11, 4


def _window_problems():
    """11 distinct problems: the c1_64 strip with its own core permittivity each, 3 modes."""
    wl, kw = mg_cases.case("c1_64")
    spec = dataclasses.replace(wl.mode_spec, num_modes=3)
    base = np.asarray(wl.eps_cross[0]).real
    core = base > base.min() + 1e-9
    out = []
    for i in range(NPROB):
        e = np.where(core, base + 0.15 * i, base).astype(complex)
        eps = [np.zeros_like(e) for _ in range(9)]
        eps[0], eps[4], eps[8] = e, e.copy(), e.copy()
        out.append(dict(eps_cross=eps, coords=wl.coords, freq=wl.freqs[0], mode_spec=spec))
    return out, kw


def _solve(problems, **kw):
    h = _cabi.Handle(max_batch=MAX_BATCH, **TOLERANCES["tight"])  # a fresh handle: no warm start from an earlier call
    try:
        return compute_modes_batch(problems, handle=h, return_info=True, **kw)
    finally:
        h.close()


def test_delivery_across_windows(built_lib):
    import torch

    problems, kw = _window_problems()
    shape = (2, 3, 64, 64, 1, 3)
    host = [np.full(shape, np.nan, complex) for _ in problems]  # pageable memory
    out_h, info_h = _solve(problems, fields_ptrs=[a.ctypes.data for a in host])
    dev = [torch.full(shape, float("nan"), dtype=torch.complex128, device="cuda") for _ in problems]
    out_d, info_d = _solve(problems, fields_ptrs=[t.data_ptr() for t in dev])
    torch.cuda.synchronize()
    for i, p in enumerate(problems):
        prob = mg_cases.model_problem(W.Workload("w", p["eps_cross"], p["coords"], np.array([p["freq"]]), p["mode_spec"]), kw)
        check_delivered(prob, "+", host[i], out_h[i][1], info_h[i]["max_residual"], "windows")
        assert np.array_equal(dev[i].cpu().numpy(), host[i]), i
        assert np.array_equal(out_d[i][1], out_h[i][1]), i
    # distinct problems: no two deliver the same n
    ns = np.array([o[1] for o in out_h])
    assert len({tuple(np.round(r.real, 12)) for r in ns}) == NPROB
    # post-processing: n unchanged, fields scaled per mode, overlaps with the previous problem across window boundaries
    out_p, info_p = _solve(problems, post=("gauge", "normalize", "flux", "overlaps"))
    coords = problems[0]["coords"]
    for i in range(NPROB):
        f_raw, f_post = host[i], out_p[i][0]
        assert np.array_equal(out_p[i][1], out_h[i][1]), i
        for m in range(3):
            a, b = f_raw[..., m].ravel(), f_post[..., m].ravel()
            c = np.vdot(a, b) / np.vdot(a, a)
            assert np.abs(b - c * a).max() <= 1e-12 * np.abs(b).max(), (i, m)
        if i > 0:
            ref = OP.dot(out_p[i - 1][0], f_post, coords)
            assert np.abs(info_p[i]["overlap_prev"] - ref).max() < 1e-9, i
    assert not info_p[0]["overlap_prev"].any()
    for i in range(MAX_BATCH, NPROB, MAX_BATCH):  # first problem of windows 2 and 3: reads the previous window's buffer
        assert np.abs(info_p[i]["overlap_prev"]).max() > 0.5, i
