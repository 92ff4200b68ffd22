"""Geometric cross-sections rasterised on the GPU (SURVEY 8(f-2)).

``ModeSolver._solver_eps(freq)`` samples the permittivity tensor of the simulation on the solver plane with nine
``Simulation.epsilon_on_grid`` calls per frequency (mode_solver.py:587-653, simulation.py:1135-1241: background value,
then every structure in order overwrites the Yee sites it contains) and hands a fresh (9,Nx,Ny) complex array to the
solver for every frequency.  That work -- and the 144 N bytes of host-to-device traffic per frequency it implies -- is
replaced by a description of WHERE the media are, which does not depend on the frequency, plus 9 numbers per medium and
frequency; ``csrc/medium.cuh::section_raster_kernel`` writes the same array straight into HBM.  Two descriptions, which
may be combined:

* primitive shapes in the solver plane: ``Rect`` (cut of a ``Box``), ``Disc`` (cut of a ``Cylinder`` along its axis or of
  a ``Sphere``), ``Polygon`` (cut of a ``PolySlab``, e.g. the trapezoid of a slanted side wall);
* ``site_medium``: a (3, Nx, Ny) integer map of the medium found at every Ex / Ey / Ez Yee site, which the caller builds
  ONCE per plane with the reference's own ``Geometry.inside_meshgrid`` (``site_medium_from_masks``): any geometry the
  reference supports, 6 bytes per cell uploaded instead of 144, nothing geometric recomputed per frequency.

    sec = Section(background=Medium(1.44**2), structures=[(Rect(center=(0, 0), size=(0.45, 0.22)), Medium(3.48**2))])
    compute_modes_batch([dict(section=sec, coords=coords, freq=f, mode_spec=spec) for f in freqs])
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _cabi


@dataclass
class Rect:
    """Cut of a ``Box`` with the solver plane: ``center`` and ``size`` in plane coordinates (geometry/base.py:1799)."""

    center: Tuple[float, float]
    size: Tuple[float, float]


@dataclass
class Disc:
    """Cut of a ``Cylinder`` whose axis is the plane normal (``dz = 0``; Cylinder.inside, geometry/primitives.py:600-632) or
    of a ``Sphere`` whose centre lies ``dz`` off the plane (Sphere.inside, primitives.py:44-70): a site is inside when
    ``|x-cx|**2 + |y-cy|**2 + dz**2 <= radius**2``."""

    center: Tuple[float, float]
    radius: float
    dz: float = 0.0


@dataclass
class Polygon:
    """Cut of a ``PolySlab``: its polygon when the slab axis is the plane normal (vertical side walls, polyslab.py:509-516),
    or the trapezoid a slab with slanted side walls shows in a plane that contains its axis.  ``vertices``: (n, 2) plane
    coordinates, either orientation, not closed.  Even-odd rule; sites exactly on an edge are unspecified (as they are in
    the reference's matplotlib ``Path.contains_points``)."""

    vertices: Sequence[Tuple[float, float]]


Shape = Union[Rect, Disc, Polygon]
SHAPE_RECT, SHAPE_DISC, SHAPE_POLYGON = 0, 1, 2

EpsLike = Union[complex, Sequence[complex], np.ndarray]


@dataclass(eq=False)
class Medium:
    """Relative permittivity of a medium: a scalar (isotropic), three numbers (diagonal, ``AnisotropicMedium``), a 3x3
    tensor (``FullyAnisotropicMedium``), or a callable ``freq -> any of those`` for dispersive media (the reference
    evaluates ``structure.eps_comp(row, col, frequency)``, simulation.py:1176-1185).  A medium is identified by the object, as
    ``Section`` does, so that it can key the per-medium dicts of ``eps_pert``: ``==`` and ``hash`` are those of the object, and
    two media with equal ``eps`` compare unequal (up to version 211 without ``eps_pert``, ``==`` compared ``eps``)."""

    eps: Union[EpsLike, Callable[[float], EpsLike]]

    def tensor(self, freq: float) -> np.ndarray:
        e = self.eps(freq) if callable(self.eps) else self.eps
        e = np.asarray(e, dtype=complex)
        if e.ndim == 0:
            return np.diag([e, e, e]).astype(complex)
        if e.shape == (3,):
            return np.diag(e).astype(complex)
        if e.shape == (3, 3):
            return e.astype(complex)
        raise ValueError("Medium.eps must be a scalar, 3 numbers or a 3x3 tensor")

    def dtensor_dfreq(self, freq: float) -> np.ndarray:
        """d eps / df (1/Hz) of the 3x3 tensor: zero for a constant medium, a central difference of ``eps(f)`` with a relative
        step of 1e-4 (error O(step^2) for a smooth model) for a dispersive one; the material term of the mode derivatives."""
        if not callable(self.eps):
            return np.zeros((3, 3), dtype=complex)
        h = 1e-4 * freq
        return (self.tensor(freq + h) - self.tensor(freq - h)) / (2 * h)

    def d2tensor_dfreq2(self, freq: float) -> np.ndarray:
        """d^2 eps / df^2 (1/Hz^2) of the 3x3 tensor: zero for a constant medium, a second central difference of ``eps(f)`` for a
        dispersive one.  The relative step is 1e-3: the roundoff of a second difference grows like eps_mach / step^2 (1e-8
        relative at 1e-4), its truncation error like step^2."""
        if not callable(self.eps):
            return np.zeros((3, 3), dtype=complex)
        h = 1e-3 * freq
        return (self.tensor(freq + h) - 2 * self.tensor(freq) + self.tensor(freq - h)) / (h * h)

    def d3tensor_dfreq3(self, freq: float) -> np.ndarray:
        """d^3 eps / df^3 (1/Hz^3) of the 3x3 tensor: zero for a constant medium, a third central difference of ``eps(f)`` at
        f +- h, f +- 2h for a dispersive one.  The relative step is 1e-3: the roundoff grows like eps_mach / step^3 (about 1e-7
        relative to eps at 1e-3), the truncation error like step^2 (exact for a cubic eps(f))."""
        if not callable(self.eps):
            return np.zeros((3, 3), dtype=complex)
        h = 1e-3 * freq
        t = self.tensor
        return (t(freq + 2 * h) - 2 * t(freq + h) + 2 * t(freq - h) - t(freq - 2 * h)) / (2 * h**3)

    def d4tensor_dfreq4(self, freq: float) -> np.ndarray:
        """d^4 eps / df^4 (1/Hz^4) of the 3x3 tensor: zero for a constant medium, a fourth central difference of ``eps(f)`` at
        f, f +- h, f +- 2h for a dispersive one.  The relative step is 5e-3: the roundoff grows like 16 eps_mach / step^4 (about 3e-6
        relative to eps at 5e-3, 1e-4 at 2e-3), the truncation error like step^2 / 6 (zero for a quartic eps(f)); the two balance
        near 5e-3."""
        if not callable(self.eps):
            return np.zeros((3, 3), dtype=complex)
        h = 5e-3 * freq
        t = self.tensor
        return (t(freq + 2 * h) - 4 * t(freq + h) + 6 * t(freq) - 4 * t(freq - h) + t(freq - 2 * h)) / h**4


def site_medium_from_masks(shape: Tuple[int, int], masks: Sequence[Tuple[np.ndarray, int]]) -> np.ndarray:
    """(3, Nx, Ny) uint16 site map from per-structure inside-masks, drawn in structure order like epsilon_on_grid
    (simulation.py:1199-1226).  ``masks``: ``(inside, medium_index)`` pairs, ``inside`` a (3, Nx, Ny) boolean array: the
    structure's ``geometry.inside_meshgrid`` evaluated at the Ex, Ey and Ez sites of the solver plane (what
    ``epsilon_on_grid`` does for the coord keys 'Ex', 'Ey', 'Ez'; the off-diagonal keys reuse the same sites,
    simulation.py:1231-1236).  Medium 0 is the background."""
    out = np.zeros((3,) + tuple(shape), dtype=np.uint16)
    for inside, idx in masks:
        inside = np.asarray(inside, dtype=bool)
        if inside.shape != out.shape:
            raise ValueError(f"inside mask has shape {inside.shape}, expected {out.shape}")
        out[inside] = idx
    return out


@dataclass
class Section:
    """``structures``: (shape, medium) pairs drawn in order on top of ``site_medium`` (when given) or of the background.
    ``media``: the media the indices of ``site_medium`` refer to (``media[0]`` must be the background); media that only
    appear in ``structures`` are appended automatically."""

    background: Medium
    structures: List[Tuple[Shape, Medium]] = field(default_factory=list)
    site_medium: Optional[np.ndarray] = None
    media: Optional[List[Medium]] = None

    def _media(self):
        media = list(self.media) if self.media is not None else [self.background]
        if media[0] is not self.background:
            raise ValueError("Section.media[0] must be the background medium")
        ids = []
        for _, m in self.structures:
            for k, known in enumerate(media):
                if known is m:
                    ids.append(k)
                    break
            else:
                media.append(m)
                ids.append(len(media) - 1)
        return media, ids

    def _site_map(self, shape):
        """The validated, contiguous uint16 site map (cached: it is the same array for every frequency of the plane)."""
        if self.site_medium is None:
            return None
        cached = getattr(self, "_site_cache", None)
        if cached is not None and cached[0] is self.site_medium:
            sm = cached[1]
        else:
            sm = np.ascontiguousarray(self.site_medium, dtype=np.uint16)
            nmedia = len(self.media) if self.media is not None else 1
            if sm.ndim != 3 or sm.shape[0] != 3:
                raise ValueError("site_medium must have shape (3, Nx, Ny): the medium at the Ex, Ey and Ez sites")
            if sm.size and int(sm.max()) >= nmedia:
                raise ValueError(f"site_medium refers to medium {int(sm.max())} but Section.media has {nmedia} entries")
            self._site_cache = (self.site_medium, sm)
        if tuple(sm.shape[1:]) != tuple(shape):
            raise ValueError("Mismatch between 'coords' and 'site_medium' shapes.")
        return sm

    def d4_table(self, freq: float) -> Optional[np.ndarray]:
        """Every medium's d^4 eps / df^4 at ``freq``, (nmedia, 9) complex128 in the order of ``pack``'s ``eps_table`` (the
        ``d4eps_table`` of b200ms_problem_ext, the material term of the fourth frequency derivative), or None when no medium is
        dispersive."""
        media, _ = self._media()
        if not any(callable(m.eps) for m in media):
            return None
        return np.ascontiguousarray([m.d4tensor_dfreq4(freq).ravel() for m in media], dtype=np.complex128)

    def pert_table(self, perts) -> np.ndarray:
        """(K, nmedia, 9) complex128 perturbation table of ``eps_pert`` (a sequence of K dicts ``{Medium: change of its eps}``, a
        scalar, three numbers or a 3x3 tensor; media not named change by 0) in the medium order of ``pack``'s ``eps_table``."""
        media, _ = self._media()
        if isinstance(perts, dict) or not isinstance(perts, (list, tuple)) or not perts or not all(isinstance(d, dict) for d in perts):
            raise ValueError("a section's eps_pert is a non-empty sequence of dicts {Medium: change of its eps}")
        table = np.zeros((len(perts), len(media), 9), dtype=np.complex128)
        for k, d in enumerate(perts):
            for m, v in d.items():
                idx = next((i for i, known in enumerate(media) if known is m), None)
                if idx is None:
                    raise ValueError("eps_pert names a medium that is not part of the section")
                if callable(v):
                    raise ValueError("eps_pert gives the change of eps at the solve's frequency: a number or a tensor, not a callable")
                table[k, idx] = Medium(v).tensor(0.0).ravel()
        return table

    def pack(self, freq: float, shape: Optional[Tuple[int, int]] = None, dispersion: bool = False, second: bool = False,
             third: bool = False):
        """ctypes ``b200ms_section`` for one frequency plus the arrays it points to (kept alive by the caller).  ``shape`` =
        (Nx, Ny) of the plane, needed to check ``site_medium``.  ``dispersion``: also pass every medium's d eps / df
        (``deps_table``), the material term of the mode derivatives; ``second``: also every medium's d^2 eps / df^2
        (``d2eps_table``), the material term of the second frequency derivative; ``third``: also every medium's d^3 eps / df^3
        (``d3eps_table``), the material term of the third frequency derivative."""
        media, ids = self._media()
        n = len(self.structures)
        rects = np.zeros((n, 4), dtype=np.float64)
        kinds = np.zeros(n, dtype=np.int32)
        pstart = np.zeros(n + 1, dtype=np.int32)
        verts = []
        for k, (g, _) in enumerate(self.structures):
            if isinstance(g, Rect):
                rects[k] = (g.center[0], g.center[1], g.size[0], g.size[1])
            elif isinstance(g, Disc):
                kinds[k] = SHAPE_DISC
                rects[k] = (g.center[0], g.center[1], g.radius, g.dz)
            elif isinstance(g, Polygon):
                v = np.asarray(g.vertices, dtype=np.float64)
                if v.ndim != 2 or v.shape[1] != 2 or v.shape[0] < 3:
                    raise ValueError("Polygon.vertices must be (n >= 3, 2)")
                kinds[k] = SHAPE_POLYGON
                verts.append(v)
            else:
                raise TypeError(f"unknown cross-section shape {type(g).__name__}")
            pstart[k + 1] = pstart[k] + (len(verts[-1]) if kinds[k] == SHAPE_POLYGON else 0)
        med = np.ascontiguousarray(ids, dtype=np.int32)
        table = np.ascontiguousarray([m.tensor(freq).ravel() for m in media], dtype=np.complex128)
        pxy = np.ascontiguousarray(np.concatenate(verts)) if verts else np.zeros((0, 2))
        site = None
        if self.site_medium is not None:
            if shape is None:
                raise ValueError("Section.pack needs the plane shape to check site_medium")
            site = self._site_map(shape)
        st = _cabi.SectionStruct()
        st.nrect = n
        st.rects = rects.ctypes.data_as(_cabi._dp)
        st.medium = med.ctypes.data_as(_cabi._ip)
        st.nmedia = len(media)
        st.eps_table = table.view(np.float64).ctypes.data_as(_cabi._dp)
        if kinds.any():
            st.shape = kinds.ctypes.data_as(_cabi._ip)
        if verts:
            st.poly_start = pstart.ctypes.data_as(_cabi._ip)
            st.poly_xy = pxy.ctypes.data_as(_cabi._dp)
        if site is not None:
            st.site_medium = site.ctypes.data_as(C.POINTER(C.c_ushort))
        dtable = None
        if dispersion and any(callable(m.eps) for m in media):
            dtable = np.ascontiguousarray([m.dtensor_dfreq(freq).ravel() for m in media], dtype=np.complex128)
            st.deps_table = dtable.view(np.float64).ctypes.data_as(_cabi._dp)
        d2table = None
        if second and any(callable(m.eps) for m in media):
            d2table = np.ascontiguousarray([m.d2tensor_dfreq2(freq).ravel() for m in media], dtype=np.complex128)
            st.d2eps_table = d2table.view(np.float64).ctypes.data_as(_cabi._dp)
        d3table = None
        if third and any(callable(m.eps) for m in media):
            d3table = np.ascontiguousarray([m.d3tensor_dfreq3(freq).ravel() for m in media], dtype=np.complex128)
            st.d3eps_table = d3table.view(np.float64).ctypes.data_as(_cabi._dp)
        return st, (rects, med, table, kinds, pstart, pxy, site, dtable, d2table, d3table)
