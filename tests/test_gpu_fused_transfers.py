"""GPU: the residual kernel that restricts its residual to the next coarser level in the same pass (transfer_vec bit 2,
csrc/march2_tma.cuh MODE_RESID_RESTRICT) gives the same bits as the separate residual and restrict4 kernels
(transfer_vec=3), and the V-cycle graph whose last sweep is redirected into the FGMRES Z slot gives the same bits as the
V-cycle run without a graph (use_graph=0, where the V-cycle writes the Z slot through its output argument).  The fused
kernel sums in restrict4_kernel's order with its contractions, so any other order or contraction shows up here as a
last-bit difference; the debug hook reports which levels took the fused kernel, so a silent fallback fails too."""
import ctypes as C

import numpy as np
import pytest

from tidy3d_b200 import _cabi
from tidy3d_b200 import workloads as W

pytestmark = pytest.mark.gpu


def _strip(nx, ny, symmetry=(0, 0), graded=False, n_core=3.48):
    eps, coords = W.strip_eps(nx, ny, n_core=n_core)
    # graded: cells from 1x to 3x the finest width, finest at the core: 3-cell aggregates and irregular lists (256 x 256 ->
    # 210 x 210 -> 117 x 117).  Shapes are ones the pair kernel covers in one strip on level 0 (multi-strip levels keep the
    # separate kernels).
    if graded:
        for a in range(2):
            n = len(coords[a]) - 1
            t = np.abs(np.linspace(-1.0, 1.0, n))
            d = 1.0 + 2.0 * t**2
            c = np.concatenate([[0.0], np.cumsum(d)])
            coords[a] = (c - c[-1] / 2) * (3.0 / c[-1])
    return W.Workload(name=f"strip_{nx}x{ny}", eps_cross=W._iso(eps), coords=coords, freqs=np.array([W.C_0 / 1.55]),
                      mode_spec=W.ModeSpecLike(num_modes=2, precision="double"), symmetry=symmetry)


def _rhs(rng, nb, nx, ny, symmetry):
    r = rng.standard_normal((nb, 2, nx, ny)) + 0j
    if symmetry[1] != 1:
        r[:, 0, :, 0] = 0  # PEC wall rows are held at zero (the V-cycle's input never has them)
    if symmetry[0] != 1:
        r[:, 1, 0, :] = 0
    return np.ascontiguousarray(r)


def _vcycles(opts, wls, r):
    """One V-cycle per problem, all problems in one device batch (b200ms_debug_batch, what = 1)."""
    pks = [_cabi.PackedProblem(w.eps_cross, w.coords, w.freqs[0], w.mode_spec, w.symmetry, "+") for w in wls]
    probs = (_cabi.Problem * len(pks))(*[p.struct for p in pks])
    h = _cabi.Handle(**opts)
    try:
        out = np.zeros_like(r)
        fused = C.c_int(-1)
        rc = _cabi.lib().b200ms_debug_batch(h._h, len(pks), probs, 1, 0, 0, _cabi._ptr(r.view(float)), None, _cabi._ptr(out.view(float)),
                                            C.byref(fused), None)
        assert rc == 0, (rc, h.last_error())
    finally:
        h.close()
    return out, fused.value


def _levels(wl):
    pk = _cabi.PackedProblem(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, wl.symmetry, "+")
    sh = (C.c_int * 40)()
    n = _cabi.lib().b200ms_debug_hierarchy(C.byref(pk.struct), None, 20, sh)
    return [(sh[2 * i], sh[2 * i + 1]) for i in range(n)]


@pytest.mark.parametrize("shape,symmetry,graded,rows", [
    ((512, 512), (0, 0), False, 0),
    ((512, 512), (1, -1), False, 0),
    ((256, 256), (-1, 1), False, 0),
    ((256, 256), (0, 0), False, 9),
    ((256, 256), (0, 0), True, 0),
    ((256, 256), (1, -1), True, 9),
])
def test_fused_residual_restriction_is_bit_identical(shape, symmetry, graded, rows):
    wl = _strip(*shape, symmetry=symmetry, graded=graded)
    assert len(_levels(wl)) >= 3
    r = _rhs(np.random.default_rng(11), 1, *shape, symmetry)
    extra = dict(stencil_pair_rows=rows) if rows else {}
    ref, fused_ref = _vcycles(dict(transfer_vec=3, **extra), [wl], r)
    new, fused = _vcycles(dict(transfer_vec=7, **extra), [wl], r)
    assert fused_ref == 0 and fused & 1, (fused_ref, fused)  # level 0 took the fused kernel, and only with bit 2
    assert np.isfinite(ref).all() and np.abs(ref).max() > 0
    assert np.array_equal(new, ref)


def test_fused_residual_restriction_batch_of_distinct_media():
    nx = ny = 256
    wls = [_strip(nx, ny, n_core=2.0 + 1.5 * i / 63) for i in range(64)]
    r = _rhs(np.random.default_rng(5), 64, nx, ny, (0, 0))
    ref, fused_ref = _vcycles(dict(transfer_vec=3), wls, r)
    new, fused = _vcycles(dict(transfer_vec=7), wls, r)
    assert fused_ref == 0 and fused & 1, (fused_ref, fused)
    assert np.isfinite(ref).all()
    assert np.array_equal(new, ref)


def test_sweep_is_the_same_with_and_without_the_fused_kernels():
    """Whole solves: the fused restriction (against transfer_vec=3) and the graph node redirected into the Z slot (against
    the ungraphed V-cycle) change no bit of the eigenvalues and fields, nor the inner iteration count."""
    from tidy3d_b200.solver import compute_modes_batch

    wl = W.si_strip(256, 2, W.sweep_freqs(4))
    problems = [dict(eps_cross=wl.eps_cross, coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec) for f in wl.freqs]
    res = {}
    for name, opts in (("separate", dict(transfer_vec=3)), ("fused", dict(transfer_vec=7)), ("no_graph", dict(use_graph=0))):
        h = _cabi.Handle(**opts)
        try:
            out = compute_modes_batch(problems, handle=h)
            res[name] = (out, h.last_stats()["inner_iters"])
        finally:
            h.close()
    a, ia = res["fused"]
    assert ia > 0
    for name in ("separate", "no_graph"):
        b, ib = res[name]
        assert ia == ib, name
        for (fa, na, _), (fb, nb, _) in zip(a, b):
            assert np.array_equal(na, nb), name
            assert np.array_equal(fa, fb), name
