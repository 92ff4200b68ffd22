"""CPU: the C-ABI library loads, exports every declared symbol, and its host-side logic (problem set-up, dense
Schur, hierarchy planning, input validation) agrees with the oracle.  No compute kernels are launched."""
import ctypes as C
import re

import numpy as np
import pytest

from oracle import restatement as R
from tests.golden.cases import CASES, resolve_kwargs


def test_abi_exports_every_declared_symbol(built_lib):
    import os

    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200ms.h")).read()
    declared = sorted(set(re.findall(r"\b(b200ms_[a-z0-9_]+)\s*\(", hdr)))
    L = built_lib.lib()
    assert set(declared) == set(built_lib.EXPORTS)
    for sym in declared:
        assert hasattr(L, sym), sym
    assert L.b200ms_version() == built_lib.ABI_VERSION == int(re.search(r"#define B200MS_VERSION (\d+)", hdr).group(1))


def test_ctypes_structs_mirror_the_header(built_lib):
    """Field order of the three ABI structs in include/b200ms.h == the ctypes mirrors (a silent mismatch would
    scramble options or results)."""
    import os

    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200ms.h")).read()

    def fields(struct_name):
        body = hdr[: hdr.index("} " + struct_name + ";")]
        body = body[body.rindex("typedef struct {") :]
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        names = []
        for decl in body.split(";"):
            m = re.search(r"(?:const\s+)?(?:double|int|long long|unsigned short|b200ms_section)\s*\*?\s*([a-z_0-9,\s\*\[\]]+)$", decl.strip())
            if m:
                for part in m.group(1).split(","):
                    names.append(re.sub(r"[\*\s]|\[\d+\]", "", part))
        return names

    for name, cls in (("b200ms_problem", built_lib.Problem), ("b200ms_result", built_lib.Result), ("b200ms_options", built_lib.Options),
                      ("b200ms_stats", built_lib.Stats), ("b200ms_section", built_lib.SectionStruct)):
        assert fields(name) == [f[0] for f in cls._fields_], name


def test_no_cpu_fallback_without_gpu(built_lib):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        built_lib.Handle()
    from tidy3d_b200 import compute_modes
    from tidy3d_b200 import workloads as W

    wl = W.c1()
    with pytest.raises(RuntimeError):
        compute_modes(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec)


def test_dense_schur(built_lib):
    L = built_lib.lib()
    rng = np.random.default_rng(0)
    for n, real in [(1, False), (2, True), (7, False), (20, True), (41, False)]:
        A = rng.standard_normal((n, n)) + (0 if real else 1j) * rng.standard_normal((n, n))
        A = np.ascontiguousarray(A.astype(complex))
        T = np.zeros((n, n), complex)
        Q = np.zeros((n, n), complex)
        rc = L.b200ms_debug_schur(n, built_lib._ptr(A.view(float)), built_lib._ptr(T.view(float)), built_lib._ptr(Q.view(float)))
        assert rc == 0
        assert np.abs(Q @ T @ Q.conj().T - A).max() < 1e-12 * max(1, np.abs(A).max()) * n
        assert np.abs(np.tril(T, -1)).max() == 0
        assert np.abs(Q.conj().T @ Q - np.eye(n)).max() < 1e-13
        ev, ev0 = np.diag(T), np.linalg.eigvals(A)
        assert np.abs(ev[:, None] - ev0[None, :]).min(axis=1).max() < 1e-10
        assert np.abs(ev[:, None] - ev0[None, :]).min(axis=0).max() < 1e-10


def _setup(built_lib, wl, kw):
    sym = kw.get("symmetry", (0, 0))
    pk = built_lib.PackedProblem(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, sym, kw.get("direction", "+"),
                                 mu_cross=kw.get("mu_cross"))
    nx, ny = pk.nx, pk.ny
    sigma = np.zeros(2)
    flags = (C.c_int * 4)()
    tgt, kn = C.c_double(), C.c_double()
    cx, cy, f = np.zeros(4 * nx, complex), np.zeros(4 * ny, complex), np.zeros((6, nx * ny), complex)
    rc = built_lib.lib().b200ms_debug_setup(
        C.byref(pk.struct), built_lib._ptr(sigma), flags, C.byref(tgt), C.byref(kn),
        built_lib._ptr(cx.view(float)), built_lib._ptr(cy.view(float)), built_lib._ptr(f.view(float)),
    )  # fmt: skip
    return rc, sigma, list(flags), tgt.value, kn.value, cx, cy, f, pk


@pytest.mark.parametrize("name", [n for n in CASES if "512" not in n and "256" not in n])
def test_host_setup_matches_oracle(built_lib, name):
    fac, kw, _ = CASES[name]
    wl = fac()
    kw = resolve_kwargs(wl, kw)
    if "split_curl_scaling" in kw:
        pytest.skip("split-curl is applied by the Python layer before the library sees the problem")
    rc, sigma, flags, tgt, kn, cx, cy, f, pk = _setup(built_lib, wl, kw)
    st = R.setup(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, kw.get("symmetry", (0, 0)), kw.get("mu_cross"))
    assert bool(flags[1]) == st["tensorial"]
    assert rc == 0
    dt = R.solver_dtype(st, "double")
    assert bool(flags[0]) == np.issubdtype(dt, np.complexfloating)
    assert abs(tgt - st["target"]) < 1e-14 and abs(kn - st["knorm"]) < 1e-14
    assert abs(sigma[0] + st["target"] ** 2) < 1e-13
    rel = lambda a, b: np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)  # noqa: E731
    assert rel(cx, np.concatenate(st["coef"][0])) < 1e-13
    assert rel(cy, np.concatenate(st["coef"][1])) < 1e-13
    e, m = st["eps"], st["mu"]
    assert rel(f, np.stack([e[0, 0], e[1, 1], e[2, 2], m[0, 0], m[1, 1], m[2, 2]])) < 1e-13


def test_hierarchy_plan(built_lib):
    from tidy3d_b200 import workloads as W

    L = built_lib.lib()
    shapes = (C.c_int * 40)()
    wl = W.si_strip(512, 4)
    pk = built_lib.PackedProblem(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec)
    n = L.b200ms_debug_hierarchy(C.byref(pk.struct), None, 20, shapes)
    got = [(shapes[2 * i], shapes[2 * i + 1]) for i in range(n)]
    assert got == [(512, 512), (256, 256), (128, 128), (64, 64), (32, 32), (16, 16), (8, 8)]
    # PML layers are not merged while they are longer than the target spacing; indefinite shift limits depth
    wl = W.c3(128)
    pk = built_lib.PackedProblem(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec)
    n = L.b200ms_debug_hierarchy(C.byref(pk.struct), None, 20, shapes)
    got = [(shapes[2 * i], shapes[2 * i + 1]) for i in range(n)]
    assert got[0] == (128, 128) and got[1][0] > 64 and all(a[0] > b[0] for a, b in zip(got, got[1:]))


def test_input_validation(built_lib):
    from tidy3d_b200 import workloads as W

    wl = W.c1()
    with pytest.raises(ValueError, match="Mismatch between 'coords' and 'esp_cross' shapes."):
        built_lib.PackedProblem(wl.eps_cross, [wl.coords[0][:-1], wl.coords[1]], wl.freqs[0], wl.mode_spec)
    with pytest.raises(ValueError, match="Wrong input to mode solver"):
        built_lib.PackedProblem(wl.eps_cross[:8], wl.coords, wl.freqs[0], wl.mode_spec)
    with pytest.raises(ValueError, match="Wrong input to mode solver"):
        built_lib.PackedProblem(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, mu_cross=wl.eps_cross[:5])


def test_section_rasterisation_host_mirror(built_lib):
    """The host mirror of section_raster_kernel (csrc/medium.cuh section_cell, shared by the device kernel) against the
    numpy restatement of epsilon_on_grid for boxes: the set-up of a `section` problem equals the set-up of the sampled
    eps_cross of the same cross-section."""
    from oracle import sections as OS
    from tidy3d_b200 import workloads as W
    from tidy3d_b200.sections import Medium, Rect, Section

    x = np.linspace(-1.0, 1.2, 24)
    y = np.cumsum(np.r_[-0.8, np.random.default_rng(3).uniform(0.04, 0.09, 30)])
    sec = Section(background=Medium(1.44**2 + 0.01j), structures=[
        (Rect((0.0, 0.1), (0.9, 0.3)), Medium([4.0, 4.2, 3.9])),
        (Rect((0.1, 0.1), (0.4, 0.2)), Medium(lambda f: 12.0 + 1e-15 * f)),
        (Rect((x[5], y[7]), (2 * (x[9] - x[5]), 2 * (y[12] - y[7]))), Medium(2.0)),  # edges exactly on Yee sites: inclusive test
    ])
    spec = W.ModeSpecLike(num_modes=2, num_pml=(3, 4))
    freq = W.C_0 / 1.3
    eps = OS.eps_on_grid(sec, [x, y], freq)
    outs = []
    for pk in (built_lib.PackedProblem(None, [x, y], freq, spec, section=sec), built_lib.PackedProblem(eps, [x, y], freq, spec)):
        nx, ny = pk.nx, pk.ny
        sigma = np.zeros(2)
        flags = (C.c_int * 4)()
        tgt, kn = C.c_double(), C.c_double()
        cx, cy, f = np.zeros(4 * nx, complex), np.zeros(4 * ny, complex), np.zeros((6, nx * ny), complex)
        rc = built_lib.lib().b200ms_debug_setup(C.byref(pk.struct), built_lib._ptr(sigma), flags, C.byref(tgt), C.byref(kn),
                                                built_lib._ptr(cx.view(float)), built_lib._ptr(cy.view(float)), built_lib._ptr(f.view(float)))
        assert rc == 0
        outs.append((sigma.copy(), list(flags), tgt.value, cx, cy, f))
    a, b = outs
    assert a[1] == b[1] and a[2] == b[2] and np.array_equal(a[0], b[0])
    assert np.array_equal(a[3], b[3]) and np.array_equal(a[4], b[4]) and np.array_equal(a[5], b[5])
    assert np.abs(b[5][0].reshape(23, 30) - eps[0]).max() < 1e-14  # exx of the set-up is the sampled eps_xx (no Jacobian here)


def _setup_of(built_lib, pk):
    nx, ny = pk.nx, pk.ny
    sigma = np.zeros(2)
    flags = (C.c_int * 4)()
    tgt, kn = C.c_double(), C.c_double()
    cx, cy, f = np.zeros(4 * nx, complex), np.zeros(4 * ny, complex), np.zeros((6, nx * ny), complex)
    rc = built_lib.lib().b200ms_debug_setup(C.byref(pk.struct), built_lib._ptr(sigma), flags, C.byref(tgt), C.byref(kn),
                                            built_lib._ptr(cx.view(float)), built_lib._ptr(cy.view(float)), built_lib._ptr(f.view(float)))
    return rc, (sigma.copy(), list(flags), tgt.value, cx, cy, f)


def _yee_sites(x, y):
    xc, yc = (x[:-1] + x[1:]) / 2, (y[:-1] + y[1:]) / 2
    return [(xc, y[:-1]), (x[:-1], yc), (x[:-1], y[:-1])]  # Ex, Ey, Ez


def test_section_shapes_and_site_map_host_mirror(built_lib):
    """Discs, polygons and the caller-made site map (b200ms_section since v201) through the host mirror of
    section_raster_kernel, against the numpy restatement of epsilon_on_grid: a fibre-like disc, a slanted-wall trapezoid, a
    concave polygon and a sphere cut, on a non-uniform grid, drawn in order over a site map that holds a slab."""
    from oracle import sections as OS
    from tidy3d_b200 import workloads as W
    from tidy3d_b200.sections import Disc, Medium, Polygon, Rect, Section, site_medium_from_masks

    rng = np.random.default_rng(11)
    x = np.cumsum(np.r_[-1.1, rng.uniform(0.03, 0.07, 44)])
    y = np.cumsum(np.r_[-0.9, rng.uniform(0.03, 0.06, 40)])
    nx, ny = x.size - 1, y.size - 1
    bg, slab, core, clad2 = Medium(1.44**2), Medium([4.0, 4.2, 3.9]), Medium(lambda f: 12.0 + 1e-15 * f), Medium(2.1 + 0.01j)
    slab_rect = Rect((0.0, -0.5), (5.0, 0.3))
    masks = np.stack([OS.inside(slab_rect, sx, sy) for sx, sy in _yee_sites(x, y)])
    site = site_medium_from_masks((nx, ny), [(masks, 1)])
    assert site.dtype == np.uint16 and 0 < site.sum() < site.size
    trapezoid = Polygon([(-0.25, -0.35), (0.25, -0.35), (0.17, -0.13), (-0.17, -0.13)])  # 70-degree side walls
    concave = Polygon([(0.5, 0.0), (0.9, 0.0), (0.9, 0.4), (0.7, 0.15), (0.5, 0.4)][::-1])  # clockwise on purpose
    sec = Section(background=bg, media=[bg, slab], site_medium=site, structures=[
        (Disc((-0.55, 0.2), 0.23), core),
        (trapezoid, core),
        (concave, clad2),
        (Disc((0.1, 0.35), 0.2, dz=0.12), clad2),  # sphere of radius 0.2 whose centre is 0.12 off the plane
        (Rect((-0.55, 0.2), (0.1, 0.1)), bg),      # a later box punches a hole into the disc
    ])
    spec = W.ModeSpecLike(num_modes=2, num_pml=(0, 0))
    freq = W.C_0 / 1.3
    eps = OS.eps_on_grid(sec, [x, y], freq)
    # the restatement really drew every shape: each medium is present, and the disc has the area of a disc
    for m in (bg, slab, core, clad2):
        assert (eps[8] == m.tensor(freq)[2, 2]).any()
    only_disc = OS.eps_on_grid(Section(background=bg, structures=[(Disc((-0.55, 0.2), 0.23), core)]), [x, y], freq)[8]
    cell_area = np.outer(np.diff(x), np.diff(y))
    assert abs(cell_area[only_disc != bg.tensor(freq)[2, 2]].sum() - np.pi * 0.23**2) < 0.1 * np.pi * 0.23**2
    rc_a, a = _setup_of(built_lib, built_lib.PackedProblem(None, [x, y], freq, spec, section=sec))
    rc_b, b = _setup_of(built_lib, built_lib.PackedProblem(eps, [x, y], freq, spec))
    assert rc_a == 0 and rc_b == 0
    assert a[1] == b[1] and a[2] == b[2] and np.array_equal(a[0], b[0])
    assert np.array_equal(a[3], b[3]) and np.array_equal(a[4], b[4]) and np.array_equal(a[5], b[5])
    assert np.abs(b[5][0].reshape(nx, ny) - eps[0]).max() < 1e-14 and np.abs(b[5][2].reshape(nx, ny) - eps[8]).max() < 1e-14


def test_section_site_map_alone_reproduces_any_sampled_geometry(built_lib):
    """A site map made from arbitrary inside-masks (here: random blobs no primitive could describe) gives exactly the array
    the reference's sampling loop would: background, then every structure's mask in order (simulation.py:1199-1226)."""
    from tidy3d_b200 import workloads as W
    from tidy3d_b200.sections import Medium, Section, site_medium_from_masks

    rng = np.random.default_rng(5)
    nx, ny = 31, 26
    x, y = np.linspace(-1, 1, nx + 1), np.linspace(-0.8, 0.8, ny + 1)
    media = [Medium(2.0), Medium(11.7 + 0.1j), Medium(np.array([[4.0, 0.1, 0], [0.1, 4.2, 0], [0, 0, 3.9]]))]
    masks = [(rng.random((3, nx, ny)) < 0.3, 1), (rng.random((3, nx, ny)) < 0.2, 2), (rng.random((3, nx, ny)) < 0.05, 0)]
    site = site_medium_from_masks((nx, ny), masks)
    freq = W.C_0 / 1.55
    want = np.zeros((9, nx, ny), complex)
    for row in range(3):
        for col in range(3):
            arr = np.full((nx, ny), media[0].tensor(freq)[row, col])
            for inside, k in masks:
                arr[inside[row]] = media[k].tensor(freq)[row, col]
            want[3 * row + col] = arr
    spec = W.ModeSpecLike(num_modes=1)
    sec = Section(background=media[0], media=media, site_medium=site)
    rc_a, a = _setup_of(built_lib, built_lib.PackedProblem(None, [x, y], freq, spec, section=sec))
    rc_b, b = _setup_of(built_lib, built_lib.PackedProblem(want, [x, y], freq, spec))
    assert rc_a == 0 and rc_b == 0 and a[1] == b[1] and a[1][1] == 1  # tensorial (off-diagonal medium)
    assert a[2] == b[2] and np.array_equal(a[0], b[0]) and np.array_equal(a[5], b[5])


def test_gpu_section_case_host_mirror_equals_restatement(built_lib):
    """The cross-section of the GPU test (tests/test_gpu_sections.py shapes_section) through the host mirror: the rasteriser
    and the restatement agree on every site, so on the GPU box only the device arithmetic is left to check; no site sits
    within 1e-9 of a shape boundary (where the reference itself is unspecified for polygons)."""
    from oracle import sections as OS
    from tests.test_gpu_sections import shapes_section
    from tidy3d_b200 import workloads as W

    sec, c = shapes_section()
    spec = W.ModeSpecLike(num_modes=3, precision="double")
    freq = float(W.sweep_freqs(3)[1])
    eps = OS.eps_on_grid(sec, [c, c], freq)
    rc_a, a = _setup_of(built_lib, built_lib.PackedProblem(None, [c, c], freq, spec, section=sec))
    rc_b, b = _setup_of(built_lib, built_lib.PackedProblem(eps, [c, c], freq, spec))
    assert rc_a == 0 and rc_b == 0 and a[1] == b[1] and np.array_equal(a[5], b[5]) and a[2] == b[2]
    import dataclasses

    for shape, _ in sec.structures:  # shrinking / growing every shape by 1e-9 must not move a site across its boundary
        for sx, sy in _yee_sites(c, c):
            if type(shape).__name__ == "Polygon":
                v = np.asarray(shape.vertices)
                ctr = v.mean(axis=0)
                lo, hi = (dataclasses.replace(shape, vertices=ctr + (v - ctr) * k) for k in (1 - 1e-8, 1 + 1e-8))
            elif type(shape).__name__ == "Disc":
                lo, hi = (dataclasses.replace(shape, radius=shape.radius * k) for k in (1 - 1e-8, 1 + 1e-8))
            else:
                lo, hi = (dataclasses.replace(shape, size=(shape.size[0] * k, shape.size[1] * k)) for k in (1 - 1e-8, 1 + 1e-8))
            assert np.array_equal(OS.inside(lo, sx, sy), OS.inside(hi, sx, sy))


def test_section_validation(built_lib):
    from tidy3d_b200 import workloads as W
    from tidy3d_b200.sections import Medium, Polygon, Rect, Section

    x = np.linspace(-1, 1, 17)
    spec = W.ModeSpecLike(num_modes=1)
    bg = Medium(2.0)
    with pytest.raises(ValueError, match="site_medium refers to medium"):
        built_lib.PackedProblem(None, [x, x], 2e14, spec, section=Section(bg, site_medium=np.ones((3, 16, 16), int)))
    with pytest.raises(ValueError, match="Mismatch between 'coords' and 'site_medium'"):
        built_lib.PackedProblem(None, [x, x], 2e14, spec, section=Section(bg, site_medium=np.zeros((3, 15, 16), int)))
    with pytest.raises(ValueError, match="Polygon.vertices"):
        built_lib.PackedProblem(None, [x, x], 2e14, spec, section=Section(bg, structures=[(Polygon([(0, 0), (1, 1)]), bg)]))
    # the library itself rejects descriptions whose indices it could not follow (B200MS_ERR_ARG), whatever the Python layer checked
    pk = built_lib.PackedProblem(None, [x, x], 2e14, spec, section=Section(bg, structures=[(Rect((0, 0), (1, 1)), Medium(3.0))]))
    pk._section_arrays[1][0] = 7  # medium index out of range
    rc, _ = _setup_of(built_lib, pk)
    assert rc == built_lib.ERR_ARG
    pk._section_arrays[1][0] = 1
    kinds = np.array([2], dtype=np.int32)  # a polygon without vertices
    pk.section.shape = kinds.ctypes.data_as(built_lib._ip)
    rc, _ = _setup_of(built_lib, pk)
    assert rc == built_lib.ERR_ARG


def test_pair_kernel_strip_geometry_covers_every_column_pair_once(built_lib):
    """Launch geometry of the pair-marching stencil kernels (csrc/march2.cuh march2_strips / march2_rows, the rule the kernels
    apply on the device restated here): every column pair of a row is an output of exactly one strip, CTA widths are whole warps,
    a row that fits one CTA has no halo pairs, and the march length is 6 m - 3 rows (the row loop is unrolled six-fold)."""
    import ctypes as C

    L = built_lib.lib()
    W, S, R = C.c_int(), C.c_int(), C.c_int()
    for ny in list(range(8, 700, 2)) + [1024, 1100, 2048, 4096, 5000]:
        assert L.b200ms_debug_march2_geometry(512, ny, 64, 264, C.byref(W), C.byref(S), C.byref(R)) == 0
        w, s, npairs = W.value, S.value, ny // 2
        assert w % 32 == 0 and 32 <= w <= 256
        owners = [0] * npairs
        for i in range(s):
            for c in range(w):
                q = i * (w - 2) + c
                if q < npairs and (c >= 1 or i == 0) and (c <= w - 2 or q == npairs - 1):
                    owners[q] += 1
        assert owners == [1] * npairs, (ny, w, s)
        if npairs <= w:
            assert s == 1
    for nx, nb, res in ((512, 64, 264), (512, 32, 264), (256, 64, 528), (128, 64, 1056), (40, 1, 264), (33, 7, 132)):
        assert L.b200ms_debug_march2_geometry(nx, 512, nb, res, C.byref(W), C.byref(S), C.byref(R)) == 0
        assert (R.value + 3) % 6 == 0 and 9 <= R.value <= 69
    # the headline level: 64 problems of 512 x 512 on 264 resident CTAs (H100: 132 SMs x 2) -> 8 CTAs of 69 rows per problem
    # = 512 CTAs, two nearly full waves
    assert L.b200ms_debug_march2_geometry(512, 512, 64, 264, C.byref(W), C.byref(S), C.byref(R)) == 0
    assert (W.value, S.value, R.value) == (256, 1, 69)
    assert L.b200ms_debug_march2_geometry(512, 511, 64, 264, C.byref(W), C.byref(S), C.byref(R)) != 0  # odd widths use the one-column kernel


def test_host_setup_matches_oracle_on_random_specs(built_lib):
    """Seeded sweep over the option space of the host set-up (csrc/host_setup.hpp: Jacobians, PML stretch, wall types, target,
    arithmetic kind, tensorial test) against the restatement, which is pinned to the reference: 1-D and 2-D planes, graded
    grids, lossy / off-diagonal / PEC-valued media, PML on either axis, both symmetry kinds, bends about either axis with either
    sign, angled planes, stated and default targets.  (200 such cases were run when this test was written.)"""
    import types

    from tidy3d_b200 import workloads as W

    rng = np.random.default_rng(20260924)
    rel = lambda a, b: np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)  # noqa: E731
    for _ in range(40):
        nx, ny = int(rng.choice([1, 12, 17, 24, 33])), int(rng.choice([1, 10, 16, 21, 30]))
        if nx == 1 and ny == 1:
            nx = 15
        x = np.cumsum(np.r_[rng.uniform(-1, 0), rng.uniform(0.03, 0.08, nx)])
        y = np.cumsum(np.r_[rng.uniform(-1, 0), rng.uniform(0.03, 0.08, ny)])
        kind = int(rng.integers(0, 4))
        base = 2.0 + 9 * rng.random((nx, ny))
        eps = [np.zeros((nx, ny), complex) for _ in range(9)]
        for k, s in zip((0, 4, 8), (1.0, 1.05, 0.95)):
            eps[k] = base * s + 0j
        if kind == 1:
            for k in (0, 4, 8):
                eps[k] = eps[k] + 1j * 0.1 * rng.random((nx, ny))
        if kind == 2:
            eps[1] = eps[3] = 0.05 * base + 0j
        if kind == 3:
            m = rng.random((nx, ny)) < 0.1
            for k in (0, 4, 8):
                eps[k][m] = -1e8
        npml = (int(rng.choice([0, 0, 3, 5])) if nx > 12 else 0, int(rng.choice([0, 0, 3, 4])) if ny > 12 else 0)
        sym = (int(rng.choice([0, 0, 1, -1])) if nx > 1 else 0, int(rng.choice([0, 0, 1, -1])) if ny > 1 else 0)
        spec = W.ModeSpecLike(num_modes=int(rng.integers(1, 4)), num_pml=npml, target_neff=None if rng.random() < 0.5 else float(rng.uniform(1.5, 3.2)))
        r = rng.random()
        if r < 0.35 and nx > 1 and ny > 1:
            spec.bend_radius, spec.bend_axis = float(rng.choice([-1, 1]) * rng.uniform(3, 10)), int(rng.integers(0, 2))
        elif r < 0.6:
            spec.angle_theta, spec.angle_phi = float(rng.uniform(-0.3, 0.3)), float(rng.uniform(-1, 1))
        wl = types.SimpleNamespace(eps_cross=eps, coords=[x, y], freqs=[W.C_0 / float(rng.uniform(1.2, 1.7))], mode_spec=spec)
        rc, sigma, flags, tgt, kn, cx, cy, f, pk = _setup(built_lib, wl, dict(symmetry=sym))
        st = R.setup(eps, [x, y], wl.freqs[0], spec, sym, None)
        ctx = (nx, ny, kind, npml, sym, vars(spec))
        assert rc == 0 and bool(flags[1]) == st["tensorial"], ctx
        assert bool(flags[0]) == np.issubdtype(R.solver_dtype(st, "double"), np.complexfloating), ctx
        assert abs(tgt - st["target"]) < 1e-13 and abs(kn - st["knorm"]) < 1e-13, ctx
        assert rel(cx, np.concatenate(st["coef"][0])) < 1e-12 and rel(cy, np.concatenate(st["coef"][1])) < 1e-12, ctx
        e, m = st["eps"], st["mu"]
        assert rel(f, np.stack([e[0, 0], e[1, 1], e[2, 2], m[0, 0], m[1, 1], m[2, 2]])) < 1e-12, ctx
