"""GPU: the pass that forms the prolongation x + P e_c and runs both post-smoothing sweeps of a V(2,2) level in one march
(transfer_vec bit 3, csrc/march2_tma.cuh MODE_PROLONG_JACOBI2) gives the same bits as the prolongation kernel followed by
two stored-diagonal sweeps (transfer_vec=7).  The pass uses the separate kernels' expressions in their order with their
contractions, so any other order or contraction shows up here as a last-bit difference; the debug hook reports which levels
took the fused pass (bits 16 + level), so a silent fallback fails too."""
import numpy as np
import pytest

from tidy3d_b200 import _cabi
from tidy3d_b200 import workloads as W

from tests.test_gpu_fused_transfers import _levels, _rhs, _strip, _vcycles

pytestmark = pytest.mark.gpu


def _post_levels(mask):
    return mask >> 16


@pytest.mark.parametrize("shape,symmetry,graded,rows", [
    ((512, 512), (0, 0), False, 0),
    ((512, 512), (1, -1), False, 0),
    ((256, 256), (-1, 1), False, 0),
    ((256, 256), (0, 0), False, 9),
    ((256, 256), (0, 0), True, 0),
    ((256, 256), (1, -1), True, 9),
])
def test_fused_post_smoothing_is_bit_identical(shape, symmetry, graded, rows):
    wl = _strip(*shape, symmetry=symmetry, graded=graded)
    assert len(_levels(wl)) >= 3
    r = _rhs(np.random.default_rng(13), 1, *shape, symmetry)
    extra = dict(stencil_pair_rows=rows) if rows else {}
    ref, mask_ref = _vcycles(dict(transfer_vec=7, **extra), [wl], r)
    new, mask = _vcycles(dict(transfer_vec=15, **extra), [wl], r)
    assert _post_levels(mask_ref) == 0 and _post_levels(mask) & 1, (mask_ref, mask)
    assert mask & 0xFFFF == mask_ref & 0xFFFF  # the residual-side fusion is unchanged
    assert np.isfinite(ref).all() and np.abs(ref).max() > 0
    assert np.array_equal(new, ref)


def test_fused_post_smoothing_batch_of_distinct_media():
    nx = ny = 256
    wls = [_strip(nx, ny, n_core=2.0 + 1.5 * i / 63) for i in range(64)]
    r = _rhs(np.random.default_rng(7), 64, nx, ny, (0, 0))
    ref, mask_ref = _vcycles(dict(transfer_vec=7), wls, r)
    new, mask = _vcycles(dict(transfer_vec=15), wls, r)
    assert _post_levels(mask_ref) == 0 and _post_levels(mask) & 1, (mask_ref, mask)
    assert np.isfinite(ref).all()
    assert np.array_equal(new, ref)


def test_fused_post_smoothing_levels():
    """On the 512^2 headline strip every explicit level (512, 256, 128; the fused tail starts at 64) takes the pass; the
    default options take it too."""
    wl = _strip(512, 512)
    levels = _levels(wl)
    assert [s[1] for s in levels[:3]] == [512, 256, 128], levels
    r = _rhs(np.random.default_rng(3), 1, 512, 512, (0, 0))
    ref, _ = _vcycles(dict(transfer_vec=7), [wl], r)
    new, mask = _vcycles({}, [wl], r)
    assert _post_levels(mask) & 0b111 == 0b111, mask
    assert np.array_equal(new, ref)


@pytest.mark.parametrize("opts,shape", [
    pytest.param({}, (256, 258), id="no_tma_ring"),  # level-0 width not a multiple of four: register pair kernel
    (dict(mg_nu=3), (256, 256)),         # V(3,3)
    ({}, (256, 1040)),                    # 520 column pairs: two strips per row on level 0
])
def test_levels_outside_the_fused_pass_keep_the_separate_kernels(opts, shape):
    wl = _strip(*shape)
    r = _rhs(np.random.default_rng(17), 1, *shape, (0, 0))
    ref, _ = _vcycles(dict(transfer_vec=7, **opts), [wl], r)
    new, mask = _vcycles(dict(transfer_vec=15, **opts), [wl], r)
    if opts:
        assert _post_levels(mask) == 0, mask
    else:
        assert not _post_levels(mask) & 1, mask  # level 0 keeps the separate kernels
    assert np.isfinite(ref).all() and np.abs(ref).max() > 0
    assert np.array_equal(new, ref)


def test_sweep_is_the_same_with_and_without_the_fused_post_smoothing():
    """Whole solves: the fused post-smoothing (default, transfer_vec=15) against the separate kernels (transfer_vec=7) and
    against the ungraphed V-cycle, whose level-0 pass writes the FGMRES Z slot through its output argument instead of the
    redirected graph node: no bit of the eigenvalues and fields changes, nor the inner iteration count."""
    from tidy3d_b200.solver import compute_modes_batch

    wl = W.si_strip(256, 2, W.sweep_freqs(4))
    problems = [dict(eps_cross=wl.eps_cross, coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec) for f in wl.freqs]
    res = {}
    for name, opts in (("fused", dict(transfer_vec=15)), ("separate", dict(transfer_vec=7)), ("no_graph", dict(use_graph=0))):
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
