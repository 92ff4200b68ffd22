"""Float64 model of the perturbation responses (derivatives "pert", "group_pert", "disp_pert"): the permittivity-gradient maps
of oracle/mode_derivatives.py, mode_group_gradient.py, mode_dispersion_gradient.py and tensor_derivatives.py contracted against
caller-given fields delta eps_k, sum over every Yee site and component of map * delta eps_k."""
import numpy as np

DIAGONAL = (0, 4, 8)  # rows xx, yy, zz of the eps_cross layout: the components a diagonal map has


def contract(grad, pert, comps=DIAGONAL):
    """grad: (ncomp, Nx, Ny) or (ncomp, Nx, Ny, M) gradient map in the rows `comps` of the eps_cross layout; pert: (K, 9, Nx, Ny)
    or (9, Nx, Ny).  Returns (K,) or (K, M)."""
    pert = np.asarray(pert, complex)
    if pert.ndim == 3:
        pert = pert[None]
    return np.einsum("axy...,kaxy->k...", np.asarray(grad), pert[:, list(comps)])


def dispersion_response(freq, d2n_dfreq_dpert, d2n_dfreq2_dpert):
    """Response of the dispersion D (ps/(nm km) per unit amplitude) to each perturbation: plugin.dispersion_of is linear in n'
    and n'', so its change is the same combination of the responses (what plugin.dispersion_gradient_of computes)."""
    from tidy3d_b200.plugin import dispersion_gradient_of

    return dispersion_gradient_of(freq, d2n_dfreq_dpert, d2n_dfreq2_dpert)
