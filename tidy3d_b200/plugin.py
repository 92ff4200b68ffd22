"""Seams into a real ``tidy3d`` install (not importable in this image: xarray/shapely/... are absent, SURVEY 8(c)).

Seam 1 (exact drop-in, one solve per call): ``tidy3d.plugins.mode.mode_solver`` imports the module-level name
``compute_modes`` (mode_solver.py:59-65) and calls it at :725 and :776; ``install()`` rebinds that name.

Seam 2 (batched, where the speed is): ``ModeSolver._solve_all_freqs(self, coords, symmetry)`` (mode_solver.py:655-672)
and ``ModeSolver._solve_all_freqs_relative(self, coords, symmetry, basis_fields)`` (:674-693) loop the single-frequency
solve over ``self.freqs``; the replacements gather ``self._solver_eps(f)`` for every frequency, run ONE device call and
reuse the reference's own ``_postprocess_solver_fields`` (:695).

Seam 2b (SURVEY 8(f-2), opt-in ``install(device_eps=True)``): instead of calling ``self._solver_eps(freq)`` -- nine
``Simulation.epsilon_on_grid`` passes over all structures and a fresh (9,Nx,Ny) complex array PER FREQUENCY
(mode_solver.py:587-653, simulation.py:1135-1241) -- ``section_of(mode_solver)`` evaluates every structure's
``geometry.inside_meshgrid`` ONCE per plane into a per-site medium map; per frequency only the 3x3 tensor of every medium is
evaluated (``Structure.eps_comp``) and the array is rasterised on the device.

Seam 3 (many mode planes, SURVEY 8(f-3)): ``run_batch(mode_solvers)`` mirrors ``tidy3d.web.api.mode.run_batch``
(web/api/mode.py:147-158) locally: the problems of ALL solvers -- including the 3x frequency copies the reference makes
for the group index (mode_solver.py:267-299) and EME cell planes (components/eme/simulation.py:521-540 build one
ModeSolver per cell) -- are collected first and solved in a single batched device call, then every ``ModeSolver.data``
is assembled by the reference's own code from the precomputed results.
"""
from __future__ import annotations

from typing import List

import numpy as np

from .solver import compute_modes, compute_modes_batch


DEVICE_EPS = False  # set by install(device_eps=True)

# plane coordinates (x', y', z' = normal) in terms of the simulation axes: what
# ModeSolver._tensorial_material_profile_modal_plane_tranform does to the rows / columns of the tensor (mode_solver.py:594-624:
# normal 0 -> swap x,y then y,z = (y, z, x); normal 1 -> swap y,z = (x, z, y))
_PLANE_AXES = {0: (1, 2, 0), 1: (0, 2, 1), 2: (0, 1, 2)}


def section_of(ms):
    """Frequency-independent description of the cross-section ``ms._solver_eps(freq)`` samples, as a
    ``tidy3d_b200.sections.Section``; ``None`` when a medium varies in space (custom media: the sampled array is needed).

    Restates the loop of ``Simulation.epsilon_on_grid`` (simulation.py:1191-1226) with the geometry part hoisted out of
    the frequency loop: background first, then ``structure.geometry.inside_meshgrid`` of every volumetric structure, in
    order, at the Ex / Ey / Ez sites of ``ms._solver_grid`` (the off-diagonal components are sampled at the site of their
    row, simulation.py:1231-1236), reduced to the plane (index 0 along the normal axis, mode_solver.py:600-601) with the
    tensor rows / columns rotated so that the normal becomes z (mode_solver.py:608-616)."""
    from .sections import Medium, Section, site_medium_from_masks

    sim, grid, normal = ms.simulation, ms._solver_grid, ms.normal_axis
    perm = _PLANE_AXES[normal]
    structures = [sim.scene.background_structure] + list(sim.volumetric_structures)
    if any(hasattr(st.medium, "eps_comp_on_grid") for st in structures):  # AbstractCustomMedium (structure.py:296-299)
        return None

    def medium_of(st):
        def tensor(freq, st=st):
            return np.array([[st.eps_comp(perm[r], perm[c], freq, None) for c in range(3)] for r in range(3)], dtype=complex)

        return Medium(tensor)

    known, media, masks = [], [], []
    site_arrays = []
    for key in ("Ex", "Ey", "Ez"):
        c = grid[key]
        site_arrays.append((np.array(c.x), np.array(c.y), np.array(c.z)))
    for k, st in enumerate(structures):
        for j, m in enumerate(known):
            if m is st.medium or m == st.medium:
                idx = j
                break
        else:
            known.append(st.medium)
            media.append(medium_of(st))
            idx = len(known) - 1
        if k == 0:
            continue  # the background fills the plane
        rows = []
        for arrays in site_arrays:
            inside = st.geometry.inside_meshgrid(*arrays)
            rows.append(np.squeeze(np.take(inside, indices=[0], axis=normal), axis=normal))
        masks.append((np.stack([rows[a] for a in perm]), idx))
    shape = masks[0][0].shape[1:] if masks else tuple(n for a, n in enumerate(len(x) for x in site_arrays[0]) if a != normal)
    return Section(background=media[0], media=media, site_medium=site_medium_from_masks(shape, masks))


def grid_correction_of(ms) -> np.ndarray:
    """``b200ms_problem.grid_correction`` table of a ``ModeSolver``: where its plane sits between the boundaries (tangential E)
    and the centres (tangential H) of the simulation grid along the plane normal -- the inputs of
    ``ModeSolver._grid_correction`` (mode_solver.py:873-883); pass it as ``grid_correction=`` with ``post=("normalize", ...)``
    so that flux normalisation and overlaps on the device include the factors the reference applies (monitor_data.py:488-503)."""
    from .postprocess import grid_correction_table

    axis, grid = ms.normal_axis, ms.simulation.grid
    return grid_correction_table(grid.boundaries.to_list[axis], grid.centers.to_list[axis], ms.plane.center[axis])


def plane_bounds_of(ms) -> np.ndarray:
    """``b200ms_problem.plane_bounds`` of a ``ModeSolver``: the extent of its plane along the two plane axes, to which the
    reference truncates the integration cells of flux and overlaps (``_diff_area`` clips to ``monitor.bounds``,
    monitor_data.py:450-455; the mode-solver monitor has the plane's centre and size, mode_solver.py to_mode_solver_monitor).
    Infinite extents stay infinite (nothing is truncated along that axis)."""
    lo, hi = (np.asarray(b, float) for b in ms.plane.bounds)
    axes = [a for a in range(3) if a != ms.normal_axis]
    return np.array([lo[axes[0]], hi[axes[0]], lo[axes[1]], hi[axes[1]]])


def _problems(ms, coords, symmetry, basis_fields=None):
    out = []
    sec = section_of(ms) if DEVICE_EPS else None
    for k, freq in enumerate(ms.freqs):
        p = dict(coords=coords, freq=freq, mode_spec=ms.mode_spec, symmetry=symmetry, direction=ms.direction)
        if sec is not None:
            p["section"] = sec  # rasterised on the device: 9 numbers per medium instead of a (9,Nx,Ny) array per frequency
        else:
            p["eps_cross"] = ms._solver_eps(freq)
        if basis_fields is not None:
            p["solver_basis_fields"] = ms._postprocess_solver_fields_inverse(basis_fields[k])  # mode_solver.py:774
        out.append(p)
    return out


def _assemble(ms, results):
    n_complex, fields, eps_spec = [], [], []
    for solver_fields, n_freq, spec in results:
        fields.append(ms._postprocess_solver_fields(solver_fields))
        n_complex.append(n_freq)
        eps_spec.append(spec)
    return n_complex, fields, eps_spec


def solve_all_freqs_batched(self, coords, symmetry):
    """Replacement body for ``ModeSolver._solve_all_freqs`` (same signature and return value)."""
    return _assemble(self, compute_modes_batch(_problems(self, coords, symmetry)))


def solve_all_freqs_relative_batched(self, coords, symmetry, basis_fields):
    """Replacement body for ``ModeSolver._solve_all_freqs_relative`` (mode_solver.py:674-693)."""
    return _assemble(self, compute_modes_batch(_problems(self, coords, symmetry, basis_fields)))


def install(batched: bool = True, device_eps: bool = None):
    """Route ``tidy3d.plugins.mode.ModeSolver`` through the CUDA library.  Raises ImportError without tidy3d.
    ``device_eps=True``: the batched seams describe each plane once by ``section_of`` and let the device rasterise the
    permittivity of every frequency (falls back to ``_solver_eps`` arrays for custom media); ``None`` keeps the setting."""
    import tidy3d.plugins.mode.mode_solver as ms  # noqa: PLC0415

    global DEVICE_EPS
    if device_eps is not None:
        DEVICE_EPS = bool(device_eps)

    ms.compute_modes = compute_modes
    ms.LOCAL_SOLVER_IMPORTED = True
    if batched:
        ms.ModeSolver._solve_all_freqs = solve_all_freqs_batched
        ms.ModeSolver._solve_all_freqs_relative = solve_all_freqs_relative_batched
    return ms.ModeSolver


class _Collected(Exception):
    """Raised by the recording pass of ``run_batch`` to leave ``ModeSolver.data`` once its problems are known."""


def run_batch(mode_solvers: List, **kwargs) -> List:
    """Local analogue of ``tidy3d.web.api.mode.run_batch(mode_solvers) -> List[ModeSolverData]`` with ONE device call for
    all planes and frequencies.

    Pass 1 runs every ``ModeSolver.data`` with ``_solve_all_freqs`` replaced by a recorder: the reference's own code
    decides coordinates, symmetry, reduced simulation copies and the extra group-index frequencies, the recorder notes the
    resulting problems and aborts.  The problems of all solvers then go to the GPU together, and pass 2 re-runs
    ``ModeSolver.data`` with ``_solve_all_freqs`` replaying the precomputed results, so everything downstream of the
    solve (colocation, normalisation, mode tracking, group index; mode_solver.py:300-343) is the reference's own code.
    """
    ModeSolver = install(batched=True)
    recorded: List[list] = []

    def record(self, coords, symmetry):
        recorded.append(_problems(self, coords, symmetry))
        raise _Collected

    saved = ModeSolver._solve_all_freqs
    ModeSolver._solve_all_freqs = record
    try:
        for ms in mode_solvers:
            try:
                ms.data  # noqa: B018  (cached_property: nothing is cached when the recorder aborts)
            except _Collected:
                pass
    finally:
        ModeSolver._solve_all_freqs = saved
    if len(recorded) != len(mode_solvers):
        raise RuntimeError("run_batch: a ModeSolver did not reach its solve (already cached?)")
    flat = [p for plist in recorded for p in plist]
    results = compute_modes_batch(flat)
    queue, pos = [], 0
    for plist in recorded:
        queue.append(results[pos : pos + len(plist)])
        pos += len(plist)

    def replay(self, coords, symmetry):
        return _assemble(self, queue.pop(0))

    ModeSolver._solve_all_freqs = replay
    try:
        return [ms.data for ms in mode_solvers]
    finally:
        ModeSolver._solve_all_freqs = saved


def group_index(n_complex, freqs, step: float):
    """Group index and dispersion from a sweep solved at the frequencies of ``ModeSolver._freqs_for_group_index``
    (``np.outer(freqs0, (1 - step, 1, 1 + step)).flatten()``, mode_solver.py:267-271), for callers that drive
    ``compute_modes_batch`` directly: the formulas of ``ModeData._group_index_post_process`` (monitor_data.py:1507-1548).
    ``n_complex``: (3 F, M).  Returns ``(freqs0, n_complex0, n_group, dispersion)`` with dispersion in ps/(nm km)."""
    n = np.asarray(n_complex).real
    f = np.asarray(freqs, float)
    back, center, fwd = n[0::3], n[1::3], n[2::3]
    f0 = f[1::3]
    inv = 1.0 / step
    n_group = center + (fwd - back) * inv * 0.5
    dispersion = (fwd * (inv + 1) + back * (inv - 1) - center * inv * 2) * f0.reshape(-1, 1) * (-1e18 * inv / C0_UM**2)
    return f0, np.asarray(n_complex)[1::3], n_group, dispersion


C0_UM = 2.99792458e14  # speed of light in um/s, the unit of the dispersion formula of monitor_data.py:1542-1548


def dispersion_of(freq, dn_dfreq, d2n_dfreq2):
    """Group-velocity dispersion (ps/(nm km)) from analytic frequency derivatives of n_eff + i k_eff
    (``compute_modes_batch(..., derivatives=("freq2",))``): D = -1e18 f^2 (2 Re n' + f Re n'') / c0^2, the step -> 0 limit of
    the three-point formula of ``group_index``.  ``freq`` broadcasts against the derivatives (e.g. shape (F, 1) with (F, M))."""
    f = np.asarray(freq, float)
    return -1e18 * f**2 * (2 * np.real(dn_dfreq) + f * np.real(d2n_dfreq2)) / C0_UM**2


def dispersion_gradient_of(freq, d2n_dfreq_deps, d2n_dfreq2_deps):
    """Permittivity gradient of the group-velocity dispersion (ps/(nm km) per unit eps) from the maps of
    ``compute_modes_batch(..., derivatives=("disp_eps",))``: -1e18 f^2 (2 Re d(n')/d eps + f Re d(n'')/d eps) / c0^2, the gradient of
    ``dispersion_of`` for a real change of eps at fixed d eps / df and d^2 eps / df^2.  ``freq`` broadcasts against the maps."""
    f = np.asarray(freq, float)
    return -1e18 * f**2 * (2 * np.real(d2n_dfreq_deps) + f * np.real(d2n_dfreq2_deps)) / C0_UM**2


def dispersion_slope_of(freq, dn_dfreq, d2n_dfreq2, d3n_dfreq3):
    """Dispersion slope S = dD / d(wavelength) (ps/(nm^2 km)) from analytic frequency derivatives of n_eff + i k_eff
    (``compute_modes_batch(..., derivatives=("freq3",))``): dD/df = -1e18 (4 f Re n' + 5 f^2 Re n'' + f^3 Re n''') / c0^2 (c0 in
    um/s) and S = -(f^2 / c) dD/df with c in nm/s, the step -> 0 limit of a central difference of ``dispersion_of`` over
    wavelength.  ``freq`` broadcasts against the derivatives like in ``dispersion_of``."""
    f = np.asarray(freq, float)
    dd = -1e18 * (4 * f * np.real(dn_dfreq) + 5 * f**2 * np.real(d2n_dfreq2) + f**3 * np.real(d3n_dfreq3)) / C0_UM**2
    return -(f**2 / (C0_UM * 1e3)) * dd


def beta3_of(freq, d2n_dfreq2, d3n_dfreq3):
    """Third-order dispersion beta3 = d^3 beta / d omega^3 (ps^3/km) of beta = omega n / c, from analytic frequency derivatives
    of n_eff + i k_eff: beta3 = (3 Re n'' + f Re n''') / (4 pi^2 c), c in m/s (1 s^3/m = 1e39 ps^3/km).  ``freq`` broadcasts
    against the derivatives like in ``dispersion_of``."""
    f = np.asarray(freq, float)
    return (3 * np.real(d2n_dfreq2) + f * np.real(d3n_dfreq3)) / (4 * np.pi**2 * (C0_UM * 1e-6)) * 1e39


def beta4_of(freq, d3n_dfreq3, d4n_dfreq4):
    """Fourth-order dispersion beta4 = d^4 beta / d omega^4 (ps^4/km) of beta = omega n / c, from analytic frequency derivatives
    of n_eff + i k_eff (``compute_modes_batch(..., derivatives=("freq4",))``): beta4 = (4 Re n''' + f Re n'''') / (8 pi^3 c), c in
    m/s (1 s^4/m = 1e51 ps^4/km).  ``freq`` broadcasts against the derivatives like in ``dispersion_of``."""
    f = np.asarray(freq, float)
    return (4 * np.real(d3n_dfreq3) + f * np.real(d4n_dfreq4)) / (8 * np.pi**3 * (C0_UM * 1e-6)) * 1e51
