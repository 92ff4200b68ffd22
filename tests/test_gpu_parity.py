"""GPU: parity of the CUDA path (through the C ABI) with the reference -- golden fixtures generated from the
unmodified reference, the oracle restatement on seeded inputs, and size-independent properties at full size."""
import os

import numpy as np
import pytest

from oracle import restatement as R
from tests.golden.cases import CASES, resolve_kwargs
from tests.helpers import (N_TOL, N_TOL_TIGHT, OVERLAP_MIN, load_golden, mode_overlaps, signature, sketch, sketch_similarity,
                           well_separated)  # fmt: skip
from tidy3d_b200 import compute_modes, compute_modes_batch
from tidy3d_b200 import workloads as W
from tidy3d_b200.solver import get_handle


def tight():
    """Handle with the "tight" tolerance preset (eig_tol 1e-9 / inner_tol 1e-10): pins n_eff to 1e-8."""
    return get_handle(tolerance="tight")

pytestmark = pytest.mark.gpu

SMALL = ["c1_64", "c1_64_minus", "c1_64_sym_pmc_pec", "lossy_48", "nonuniform_56", "slab1d_x1", "slab1d_y1",
         "c3_96", "c4_96", "c4_96_axis0", "strip_128_m4", "c3_128", "c4_128",
         "angled_64", "angled_48_minus", "angled_phi_48", "offdiag_48", "pec_block_40", "lossy_angled_40", "lossy_angled_40_minus", "angle_bend_44",
         "mu_cross_40", "split_curl_40", "pec_split_40"]  # fmt: skip
LARGE = ["c2_256_f0", "headline_512_f0", "c3_512", "c4_512"]


def _solve(name, preset="reference"):
    fac, kw, _ = CASES[name]
    wl = fac()
    kw = resolve_kwargs(wl, kw)
    out, info = compute_modes_batch(
        [dict(eps_cross=wl.eps_cross, coords=wl.coords, freq=wl.freqs[0], mode_spec=wl.mode_spec, **kw)], return_info=True,
        handle=get_handle(tolerance=preset),
    )
    return wl, out[0], info[0]


def _check_against_golden(name, fields, n, spec, preset):
    g = load_golden(name)
    assert spec == str(g["spec"])
    # tolerances stated in DESIGN.md section 6.  Library default ("reference" preset == the reference's own ARPACK
    # tolerance): |dn_eff|, |dk_eff| <= 1e-6 against the reference run at that tolerance AND against the reference re-run
    # with TOL_EIGS = 1e-12.  "tight" preset: <= 1e-8 against the latter.
    assert np.abs(n - g["n_ref"]).max() < N_TOL
    assert np.abs(n - g["n_tight"]).max() < (N_TOL_TIGHT if preset == "tight" else N_TOL)
    if "fields_tight" in g.files:
        ok = well_separated(g["n_tight"])
        ov = mode_overlaps(fields, g["fields_tight"])  # E and H blocks separately + their relative phase
        # |eps| = 1e8 inside metal amplifies the eigenvector error at the reference's own (loose) tolerance
        ov_min = 0.99 if ("pec" in name and preset == "reference") else OVERLAP_MIN
        assert (ov[ok] > ov_min).all(), ov
    # per-mode component amplitudes |E_x|..|H_z| (phase independent; catches a wrong H scale or a dropped component);
    # each block is compared relative to its own largest component
    sig, ref = signature(fields), g["sig_tight"]
    ok = well_separated(g["n_tight"])
    tol = 2e-6 if preset == "tight" else 1e-3
    if "pec" in name:
        # |eps| = 1e8 in the metal amplifies the eigenvector error there (max_residual ~ 2e-4 even with the tight preset); at
        # the reference's tolerance the small H_z of a mode is good to a few per cent of the mode's largest H component
        tol = 1e-3 if preset == "tight" else 0.1
    for blk in (slice(0, 3), slice(3, 6)):
        err = np.abs(sig[:, blk] - ref[:, blk]) / ref[:, blk].max(axis=1, keepdims=True)
        assert err[ok].max() < tol, (name, err)


@pytest.mark.parametrize("preset", ["reference", "tight"])
@pytest.mark.parametrize("name", SMALL)
def test_golden_small(name, preset):
    wl, (fields, n, spec), info = _solve(name, preset)
    assert fields.shape == (2, 3, wl.eps_cross[0].shape[0], wl.eps_cross[0].shape[1], 1, wl.mode_spec.num_modes)
    assert fields.dtype == np.complex128 and info["converged"] == wl.mode_spec.num_modes
    _check_against_golden(name, fields, n, spec, preset)


# inner (FGMRES) iterations per shift-invert apply with the library defaults, measured on an H100 80GB HBM3 (400 W limit).
# The eigenpairs do not depend on the preconditioner, so a multigrid that has gone subtly wrong shows up only here, as more
# inner iterations (tests/test_gpu_kernels_vs_model.py pins the kernels themselves).
INNER_PER_APPLY = {"c1_64": 262 / 38, "c3_128": 906 / 62, "c4_128": 1128 / 44, "lossy_48": 353 / 47, "angled_64": 1003 / 100}


@pytest.mark.parametrize("name", sorted(INNER_PER_APPLY))
def test_inner_iterations_per_apply_stay_in_budget(name):
    _, _, info = _solve(name)
    assert info["op_applies"] > 0
    assert info["inner_iters"] / info["op_applies"] <= 1.3 * INNER_PER_APPLY[name], info


@pytest.mark.parametrize("preset", ["reference", "tight"])
@pytest.mark.parametrize("name", LARGE)
def test_golden_full_size(name, preset):
    """BASELINE.json configs at their full grid sizes (n_complex and field signatures pinned by the unmodified reference)."""
    wl, (fields, n, spec), info = _solve(name, preset)
    _check_against_golden(name, fields, n, spec, preset)
    assert info["max_residual"] < (1e-5 if preset == "tight" else 1e-3)
    # full-size FIELD parity: a seeded 16-vector random sketch of the reference's fields (TOL_EIGS = 1e-12) is committed
    # instead of the 50-100 MB arrays (tests/golden/make_sketch_golden.py); similarity = 1 - O(err^2) up to each mode's phase
    path = os.path.join(os.path.dirname(__file__), "golden", name + "_sketch.npz")
    if os.path.exists(path):
        g = np.load(path)
        ok = well_separated(g["n_tight"])
        sim = sketch_similarity(sketch(fields), g["sketch"])
        assert (sim[ok] > (1 - 1e-8 if preset == "tight" else 1 - 1e-4)).all(), (name, 1 - sim)


SINGLE = ["c1_64_single", "c3_96_single", "c4_96_single", "lossy_48_single", "angled_64_single"]


@pytest.mark.parametrize("name", SINGLE)
def test_golden_single_precision(name):
    """mode_spec.precision = "single" -- the reference's default (components/mode.py:105-106).  The reference then solves a
    float32/complex64 eigenproblem with trimmed entries (solver.py:396-420, 497-498) and returns complex64 fields; its own
    single and double results differ by up to 5e-6 in n (fixtures: max|n_ref - n_tight|).  Contract (DESIGN.md section 6):
    complex64 fields, |n - n_single_ref| <= 2e-5, |n - n_double_ref| <= 1e-6 (we solve in fp64), E/H overlaps >= 0.999
    against the reference's own single-precision fields."""
    wl, (fields, n, spec), info = _solve(name)
    g = load_golden(name)
    assert fields.dtype == np.complex64 and spec == str(g["spec"])
    assert np.abs(n - g["n_ref"]).max() < 2e-5
    assert np.abs(n - g["n_tight"]).max() < N_TOL
    ok = well_separated(g["n_tight"])
    ov = mode_overlaps(fields.astype(complex), g["fields_ref"].astype(complex))
    assert (ov[ok] > OVERLAP_MIN).all(), ov


def test_reference_compute_modes_smoke_input():
    """The reference's own direct test of compute_modes (tests/test_plugins/test_mode_solver.py:170-181): random 10x10
    array used for all nine tensor components, direction "-", default single precision.  That test asserts nothing but
    "returns"; the input is pathological (singular tensor: every Schur-complement entry of eps is zero) and the reference
    itself fails on it with ArpackNoConvergence for some seeds and at tighter tolerances (tests/golden/make_golden.py).
    Mirrored contract: the call returns arrays of the documented shapes/dtypes and eps_spec, or raises the documented
    no-convergence RuntimeError -- never garbage, never a crash."""
    for name, dt in (("rand10_single", np.complex64), ("rand10_double", np.complex128)):
        fac, kw, _ = CASES[name]
        wl = fac()
        try:
            f, n, spec = compute_modes(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, **kw)
        except RuntimeError as e:
            assert "did not converge" in str(e)
            continue
        assert f.shape == (2, 3, 10, 10, 1, 3) and f.dtype == dt and spec == "tensorial_real"
        assert np.isfinite(f).all() and np.isfinite(n).all()


def test_pml_with_default_target_cluster():
    """PML + target_neff=None at 128^2 (SURVEY 7.3 hard part 3): two PML modes with k_eff ~ 0.74 that differ by 1e-5 in n
    are among the four wanted; the reference needs ~1400 OP applies.  n_complex to the stated tolerances, single modes by
    overlap, the near-degenerate pair by the principal angle between the two-dimensional subspaces."""
    from tests.helpers import cluster_overlaps

    for preset, tol in (("reference", N_TOL), ("tight", 1e-7)):
        wl, (fields, n, spec), info = _solve("pml_none_128", preset)
        g = load_golden("pml_none_128")
        assert np.abs(n - g["n_ref"]).max() < tol and np.abs(n - g["n_tight"]).max() < tol
        for members, smin in cluster_overlaps(fields, g["fields_tight"].astype(complex), g["n_tight"], gap=1e-4):
            assert smin > 0.99, (members, smin)


def test_against_oracle_seeded_random_sections():
    """Random (seeded) smooth cross-sections: CUDA path vs the oracle restatement run side by side."""
    rng = np.random.default_rng(1234)
    for trial in range(3):
        nx, ny = int(rng.integers(30, 60)), int(rng.integers(30, 60))
        x = np.linspace(-1.2, 1.2, nx + 1)
        y = np.linspace(-1.0, 1.0, ny + 1)
        xm, ym = 0.5 * (x[:-1] + x[1:]), 0.5 * (y[:-1] + y[1:])
        blob = np.exp(-((xm[:, None] / 0.35) ** 2) - ((ym[None, :] - 0.1) / 0.25) ** 2)
        base = 2.1 + 8.0 * blob + 0.2 * rng.random((nx, ny))
        eps = [np.zeros((nx, ny), complex) for _ in range(9)]
        eps[0], eps[4], eps[8] = base + 0j, 1.05 * base + 0j, 0.95 * base + 0j
        spec = W.ModeSpecLike(num_modes=3, num_pml=(0, 6) if trial == 1 else (0, 0), target_neff=None if trial < 2 else 2.2)
        f, n, s = compute_modes(eps, [x, y], W.C_0 / 1.31, spec, handle=tight())
        f0, n0, s0 = R.compute_modes(eps, [x, y], W.C_0 / 1.31, spec, tol=1e-12)
        assert s == s0
        assert np.abs(n - n0).max() < 1e-8
        ok = well_separated(n0)
        assert (mode_overlaps(f, f0)[ok] > OVERLAP_MIN).all()


def test_frequency_batch_equals_single_solves():
    """Batched sweep (one device call) == independent solves; also pins two sweep points to the oracle."""
    wl = W.c2(nf=6, n=96)
    probs = [dict(eps_cross=wl.eps_cross, coords=wl.coords, freq=f, mode_spec=wl.mode_spec) for f in wl.freqs]
    batch = compute_modes_batch(probs, handle=tight())
    for i in (0, 5):
        f1, n1, _ = compute_modes(wl.eps_cross, wl.coords, wl.freqs[i], wl.mode_spec, handle=tight())
        assert np.abs(batch[i][1] - n1).max() < 1e-9
        assert (mode_overlaps(batch[i][0], f1) > 1 - 1e-6).all()
        _, n0, _ = R.compute_modes(wl.eps_cross, wl.coords, wl.freqs[i], wl.mode_spec, tol=1e-12)
        assert np.abs(batch[i][1] - n0).max() < 1e-8
    ns = np.array([b[1] for b in batch])
    assert (np.diff(ns[:, 0].real) < 0).all()  # n_eff falls with wavelength along the sweep


def test_c5_planes_batch_distinct_cross_sections():
    """BASELINE config 5 in miniature: several mode planes (different core widths) x frequencies in ONE batch, so
    the problems of a device batch carry different coefficient fields (no sharing)."""
    planes = W.c5_planes(n_planes=3, n=64, nf=2)
    probs = [dict(eps_cross=p.eps_cross, coords=p.coords, freq=f, mode_spec=p.mode_spec) for p in planes for f in p.freqs]
    out = compute_modes_batch(probs, handle=tight())
    assert len(out) == 6
    for pr, (f, n, s) in zip(probs, out):
        _, n0, _ = R.compute_modes(pr["eps_cross"], pr["coords"], pr["freq"], pr["mode_spec"], tol=1e-12)
        assert np.abs(n - n0).max() < 1e-8
    widths_n1 = [out[2 * i][1][0].real for i in range(3)]
    assert widths_n1[0] < widths_n1[1] < widths_n1[2]  # wider core -> larger fundamental n_eff


def test_mixed_batch_groups_and_ragged_inputs():
    """One call with different grid sizes, arithmetic kinds and mode counts; and an empty batch."""
    assert compute_modes_batch([]) == []
    names = ["c1_64", "lossy_48", "slab1d_x1", "c1_64_sym_pmc_pec"]
    probs, refs = [], []
    for name in names:
        fac, kw, _ = CASES[name]
        wl = fac()
        probs.append(dict(eps_cross=wl.eps_cross, coords=wl.coords, freq=wl.freqs[0], mode_spec=wl.mode_spec, **kw))
        refs.append(load_golden(name)["n_tight"])
    out = compute_modes_batch(probs, handle=tight())
    for (f, n, s), nref in zip(out, refs):
        assert np.abs(n - nref).max() < 1e-8


def test_n_complex_only_mode():
    """want_fields=False: only n_complex is produced (no epilogue kernel, no field transfer)."""
    wl = W.c1()
    probs = [dict(eps_cross=wl.eps_cross, coords=wl.coords, freq=f, mode_spec=wl.mode_spec) for f in (wl.freqs[0], 1.02 * wl.freqs[0])]
    out = compute_modes_batch(probs, want_fields=False, handle=tight())
    assert out[0][0] is None and out[0][2] == "diagonal"
    assert np.abs(out[0][1] - load_golden("c1_64")["n_tight"]).max() < 1e-8
    assert out[1][1][0].real > out[0][1][0].real  # higher frequency -> larger n_eff


def test_direction_and_precision_contract():
    wl = W.c1()
    fp, n_p, _ = compute_modes(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, direction="+")
    fm, n_m, _ = compute_modes(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, direction="-")
    assert np.abs(n_p - n_m).max() < 1e-10
    sign = np.ones((2, 3, 1, 1, 1, 1))
    sign[1, 0] = sign[1, 1] = sign[0, 2] = -1  # solver.py:370-373
    for m in range(2):
        ph = np.vdot(fp[0, 0, ..., m].ravel(), fm[0, 0, ..., m].ravel())
        ph /= abs(ph)
        assert np.abs(fm[..., m] - ph * (sign[..., 0] * fp[..., m])).max() < 1e-6 * np.abs(fp[..., m]).max()
    wl.mode_spec.precision = "single"
    fs, n_s, _ = compute_modes(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec)
    assert fs.dtype == np.complex64  # solver.py:265-267
    assert np.abs(n_s - n_p).max() < 1e-5


def test_relative_mode_solver_matches_reference():
    """solver_basis_fields path (solver_eigs_relative, solver.py:750-776) against a fixture made by the reference."""
    from tests.golden.cases import relative_case

    wl = relative_case()
    g = load_golden("relative_48")
    f, n, spec = compute_modes(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, solver_basis_fields=g["basis"])
    assert spec == "diagonal"
    assert np.abs(n - g["n_ref"]).max() < 1e-9
    assert (mode_overlaps(f, g["fields_tight"]) > 1 - 1e-8).all()
    with pytest.raises(ValueError, match="Shape mismatch between 'basis_fields'"):
        compute_modes(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, solver_basis_fields=g["basis"][..., :2])


def test_edge_shapes_and_mode_counts():
    """Tiny and odd-sized grids, one mode, many modes (ncv grows with k like scipy's max(2k+1, 20))."""
    rng = np.random.default_rng(7)
    for (nx, ny, k) in [(10, 10, 2), (33, 47, 1), (61, 29, 3), (40, 40, 11)]:
        x = np.linspace(-1.0, 1.0, nx + 1)
        y = np.linspace(-0.8, 0.8, ny + 1)
        xm, ym = 0.5 * (x[:-1] + x[1:]), 0.5 * (y[:-1] + y[1:])
        base = 2.0 + 9.0 * np.exp(-((xm[:, None] / 0.3) ** 2) - (ym[None, :] / 0.2) ** 2) + 0.05 * rng.random((nx, ny))
        eps = [np.zeros((nx, ny), complex) for _ in range(9)]
        eps[0], eps[4], eps[8] = base + 0j, base + 0j, base + 0j
        spec = W.ModeSpecLike(num_modes=k)
        f, n, s = compute_modes(eps, [x, y], W.C_0 / 1.55, spec, handle=tight())
        f0, n0, s0 = R.compute_modes(eps, [x, y], W.C_0 / 1.55, spec, tol=1e-12)
        assert f.shape == (2, 3, nx, ny, 1, k) and s == s0
        assert np.abs(n - n0).max() < 1e-8, (nx, ny, k, np.abs(n - n0).max())


def test_incidence_matrix_branch_with_mu_cross():
    """PEC cells together with mu_cross: the reference switches to its incidence-matrix formulation (solver.py:93, 441-449,
    474-477, 506-508, 568-569: PEC unknowns removed, 1/eps_zz zeroed).  No committed fixture for this combination: the
    CUDA path is compared with the oracle restatement run side by side (the split-curl twin is the golden pec_split_40)."""
    fac, kw, _ = CASES["pec_block_40"]
    wl = fac()
    n = wl.eps_cross[0].shape[0]
    mu = [np.zeros((n, n), complex) for _ in range(9)]
    yy = np.broadcast_to(np.arange(n)[None, :] < n // 3, (n, n))
    mu[0], mu[4], mu[8] = 1.0 + 0.3 * yy + 0j, 1.0 + 0.2 * yy + 0j, 1.0 + 0.1 * yy + 0j
    f, nn, s = compute_modes(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, mu_cross=mu, handle=tight())
    f0, n0, s0 = R.compute_modes(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, mu_cross=mu, tol=1e-12)
    assert s == s0 and np.abs(nn - n0).max() < 1e-8
    assert (mode_overlaps(f, f0)[well_separated(n0)] > OVERLAP_MIN).all()
    metal = np.abs(np.asarray(wl.eps_cross[0])) >= 0.9e8
    assert np.abs(f[0, 0][metal]).max() == 0.0  # removed unknowns come back as exact zeros (solver.py:568-569)


def test_full_size_properties_headline_batch():
    """Size-independent checks at the headline size on a multi-frequency batch: true eigen-residuals, unit-norm
    eigenvectors, H/E consistency of the recovered fields (Hz = (Dxf Ey - Dyf Ex) recomputed on the host)."""
    wl = W.headline(nf=4)
    probs = [dict(eps_cross=wl.eps_cross, coords=wl.coords, freq=f, mode_spec=wl.mode_spec) for f in wl.freqs]
    out, info = compute_modes_batch(probs, return_info=True, handle=tight())
    g = load_golden("headline_512_f0")
    assert np.abs(out[0][1] - g["n_tight"]).max() < 1e-8
    for (f, n, _), inf, freq in zip(out, info, wl.freqs):
        assert inf["converged"] == 4 and inf["max_residual"] < 1e-5
        ex, ey, hz = f[0, 0, :, :, 0, :], f[0, 1, :, :, 0, :], f[1, 2, :, :, 0, :]
        nrm = np.sqrt((np.abs(ex) ** 2 + np.abs(ey) ** 2).sum(axis=(0, 1)))
        assert np.allclose(nrm, 1.0, atol=1e-9)
        k0 = 2 * np.pi * freq / W.C_0
        dl = wl.coords[0][1] - wl.coords[0][0]
        dxf_ey = np.zeros_like(ey)
        dxf_ey[:-1] = (ey[1:] - ey[:-1]) / dl
        dxf_ey[-1] = -ey[-1] / dl
        dxf_ey[0] = ey[1] / dl  # PEC row (derivatives.py:15-16)
        dyf_ex = np.zeros_like(ex)
        dyf_ex[:, :-1] = (ex[:, 1:] - ex[:, :-1]) / dl
        dyf_ex[:, -1] = -ex[:, -1] / dl
        dyf_ex[:, 0] = ex[:, 1] / dl
        hz_ref = (dxf_ey - dyf_ex) / k0 * (-1j / R.ETA_0)
        assert np.abs(hz - hz_ref).max() < 1e-9 * np.abs(hz_ref).max() + 1e-12
